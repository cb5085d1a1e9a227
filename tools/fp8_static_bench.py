"""Static-scale FP8 U-Net measurement: fusion_precision 'bf16', 'fp8' and 'fp8_static' on the vitl 4K P49 workload
(cai_mode m2, process_num 9, synthetic weights), in alternated timed windows.

    python tools/fp8_static_bench.py --out DIR [--steps 3] [--windows 3] [--calib-images 2]

The 'fp8_static' model is calibrated first (PatchFusion.calibrate_fp8, m2) on --calib-images seeded random 4K images
that are not the timed one.  Writes DIR/fp8_static_bench.json and prints it:
  * gpu: card name and power limit (nvidia-smi, in the same process), median SM clock over the timed windows;
  * tiles/s of each model per window and the median, launches per step;
  * per-step ms from the library's per-launch CUDA events over --steps profiled steps: the E4M3 convs (per-tile and
    static kernels), the static quantize launches and the per-tile amax / quantize launches;
  * depth: max-abs / mean-abs difference of 'fp8_static' from 'bf16' and from 'fp8' on the timed image.
"""
import argparse
import json
import os
import random
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from fp8_bench import gpu_info   # noqa: E402

KINDS = {'pf_conv3_halo_e4m3_kernel': 'e4m3_conv_tiles', 'pf_conv3_halo_e4m3_q8_kernel': 'e4m3_conv_static',
         'quant_static_kernel': 'quantize_static', 'quant_amax_kernel': 'amax', 'quant_write_kernel': 'quantize_tiles',
         'pf_conv3_halo_kernel': 'bf16_halo_conv'}


def profile(model, lr, img, steps):
    from patchfusion_b200 import lib
    per = []
    for _ in range(steps):
        prof = lib.Profiler()
        lib.PROFILER = prof
        try:
            prof.start()
            model(mode='infer', image_lr=lr, image_hr=img, cai_mode='m2', process_num=9)
            recs = prof.stop()
        finally:
            lib.PROFILER = None
        d = {k: 0.0 for k in KINDS.values()}
        for name, label, flops, ms in recs:
            if name in KINDS:
                d[KINDS[name]] += ms
        per.append(d)
    return {k: round(statistics.median(x[k] for x in per), 3) for k in per[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--windows', type=int, default=3)
    ap.add_argument('--calib-images', type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('fp8_static_bench: no CUDA device (the measurement runs on the GPU only)')
    os.makedirs(args.out, exist_ok=True)
    import bench
    from patchfusion_b200 import lib
    from patchfusion_b200.model import PatchFusion
    gpu = gpu_info()
    dev = torch.device('cuda')
    cfg, sd = bench.build_inputs('vitl')
    models = {}
    for prec in ('bf16', 'fp8', 'fp8_static'):
        m = PatchFusion(dict(cfg, fusion_precision=prec))
        m.load_state_dict(sd, strict=True)
        models[prec] = m.to(dev).eval()
    cal = torch.rand(args.calib_images, 3, 2160, 3840, generator=torch.Generator().manual_seed(1234)).to(dev)
    random.seed(0)
    table = models['fp8_static'].calibrate_fp8(models['fp8_static'].make_lr(cal), cal, cai_mode='m2', process_num=9)
    del cal
    img = torch.rand(1, 3, 2160, 3840, generator=torch.Generator().manual_seed(7)).to(dev)
    lr = models['bf16'].make_lr(img)

    def step(m):
        return m(mode='infer', image_lr=lr, image_hr=img, cai_mode='m2', process_num=9)[0]

    outs = {}
    for prec, m in models.items():
        for _ in range(3):
            outs[prec] = step(m).clone()
    torch.cuda.synchronize()

    def diff(a, b):
        d = (outs[a] - outs[b]).abs()
        return dict(max_abs=d.max().item(), mean_abs=d.mean().item())
    depth = dict(fp8_static_vs_bf16=diff('fp8_static', 'bf16'), fp8_static_vs_fp8=diff('fp8_static', 'fp8'),
                 fp8_vs_bf16=diff('fp8', 'bf16'), bf16_range=[outs['bf16'].min().item(), outs['bf16'].max().item()])

    sampler = bench.ClockSampler(torch.cuda.current_device())
    res = {p: [] for p in models}
    launches = {}
    for _ in range(args.windows):
        for prec, m in models.items():
            torch.cuda.synchronize()
            l0 = lib.launch_count() + m.graph_launches
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                step(m)
            e1.record()
            torch.cuda.synchronize()
            launches[prec] = (lib.launch_count() + m.graph_launches - l0) // args.steps
            res[prec].append(49 * args.steps / (e0.elapsed_time(e1) / 1e3))
    clocks = sampler.stop()
    out = dict(
        gpu=dict(gpu, median_sm_clock_mhz=clocks.get('sm_mhz'), clock_reasons=clocks.get('reasons')),
        workload='Depth-Anything-vitl PatchFusion, 4K P49, cai_mode m2, process_num 9, synthetic weights',
        tiles_per_s={p: [round(x, 2) for x in v] for p, v in res.items()},
        median_tiles_per_s={p: round(statistics.median(v), 2) for p, v in res.items()},
        launches_per_step=launches,
        per_step_ms={p: profile(m, lr, img, args.steps) for p, m in models.items()},
        depth=depth, calibration_table=table)
    p = os.path.join(args.out, 'fp8_static_bench.json')
    with open(p, 'w') as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
