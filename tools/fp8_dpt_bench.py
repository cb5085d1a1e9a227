"""Static-scale FP8 DPT decoder measurement: (vit, fusion, dpt) precisions {bf16 / bf16 / bf16, bf16 / bf16 / fp8_static,
fp8_static / fp8_static / bf16, fp8_static / fp8_static / fp8_static} on the vitl 4K P49 workload (cai_mode m2,
process_num 9, synthetic weights), in alternated timed windows.

    python tools/fp8_dpt_bench.py --out DIR [--steps 3] [--windows 3] [--calib-images 2]

The FP8 models are calibrated first (PatchFusion.calibrate_fp8, m2) on --calib-images seeded random 4K images that are
not the timed one.  A model's workspaces and graphs are released after each of its windows and rebuilt by two untimed
steps before the next (four vitl 4K models do not fit in 80 GB with theirs).  Writes DIR/fp8_dpt_bench.json and
prints it:
  * gpu: card name and power limit (nvidia-smi, in the same process), median SM clock over the timed windows;
  * tiles/s of each model per window, the median and the spread (max - min), launches per step;
  * per-step ms from the library's per-launch CUDA events over --steps profiled steps: the DPT decoders' 19 covered
    convs per branch call (the 3x3 convs of N = C or C / 2 between a branch call's patch gather and its metric-bins
    tail: a branch has no other such conv) and every static quantize launch (in the DPT-only arm these are the DPT's
    five per branch call);
  * depth: max-abs / mean-abs difference of each FP8 model from bf16 on the timed image.
"""
import argparse
import json
import os
import random
import re
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

from fp8_bench import gpu_info   # noqa: E402
from fp8_vit_bench import release   # noqa: E402

MODELS = {'bf16': {}, 'dpt_fp8_static': dict(dpt_precision='fp8_static'),
          'vit_unet_fp8_static': dict(vit_precision='fp8_static', fusion_precision='fp8_static'),
          'all_fp8_static': dict(vit_precision='fp8_static', fusion_precision='fp8_static', dpt_precision='fp8_static')}
LABEL_RE = re.compile(r'rows(\d+) K(\d+)x(\d+) N(\d+)')


def is_dpt_conv(label, C):
    """a covered DPT conv's profiler label, given that the launch is inside a branch call"""
    m = LABEL_RE.search(label)
    return bool(m) and label.startswith('conv3x3') and int(m.group(2)) == 9 and int(m.group(4)) in (C, C // 2)


def profile(model, lr, img, steps, C):
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
        d = dict(dpt_convs_ms=0.0, dpt_convs_launches=0, quant_static_ms=0.0, quant_static_launches=0)
        in_branch = False
        for name, label, flops, ms in recs:
            if name == 'patch_im2col_kernel':
                in_branch = True
            elif name == 'logbinom_depth_kernel':
                in_branch = False
            if in_branch and is_dpt_conv(label, C):
                d['dpt_convs_ms'] += ms
                d['dpt_convs_launches'] += 1
            if name == 'quant_static_kernel':
                d['quant_static_ms'] += ms
                d['quant_static_launches'] += 1
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
        raise SystemExit('fp8_vit_bench: no CUDA device (the measurement runs on the GPU only)')
    os.makedirs(args.out, exist_ok=True)
    import bench
    from patchfusion_b200 import lib
    from patchfusion_b200.model import PatchFusion
    gpu = gpu_info()
    dev = torch.device('cuda')
    cfg, sd = bench.build_inputs('vitl')
    from patchfusion_b200.params import branch_hparams
    C = branch_hparams(cfg['fine_branch'])['features']
    models = {}
    for name, kw in MODELS.items():
        m = PatchFusion(dict(cfg, **kw))
        m.load_state_dict(sd, strict=True)
        models[name] = m.to(dev).eval()
    cal = torch.rand(args.calib_images, 3, 2160, 3840, generator=torch.Generator().manual_seed(1234)).to(dev)
    for name, m in models.items():
        if name != 'bf16':
            random.seed(0)
            m.calibrate_fp8(m.make_lr(cal), cal, cai_mode='m2', process_num=9)
            release(m)
    del cal
    img = torch.rand(1, 3, 2160, 3840, generator=torch.Generator().manual_seed(7)).to(dev)
    lr = models['bf16'].make_lr(img)

    def step(m):
        return m(mode='infer', image_lr=lr, image_hr=img, cai_mode='m2', process_num=9)[0]

    outs = {}
    for name, m in models.items():
        for _ in range(3):
            outs[name] = step(m).clone()
        release(m)

    def diff(a, b):
        d = (outs[a] - outs[b]).abs()
        return dict(max_abs=d.max().item(), mean_abs=d.mean().item())
    depth = {'%s_vs_bf16' % n: diff(n, 'bf16') for n in models if n != 'bf16'}
    depth['bf16_range'] = [outs['bf16'].min().item(), outs['bf16'].max().item()]

    sampler = bench.ClockSampler(torch.cuda.current_device())
    res = {n: [] for n in models}
    launches = {}
    for _ in range(args.windows):
        for name, m in models.items():
            for _ in range(2):                      # untimed: workspaces and graphs back
                step(m)
            torch.cuda.synchronize()
            l0 = lib.launch_count() + m.graph_launches
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                step(m)
            e1.record()
            torch.cuda.synchronize()
            launches[name] = (lib.launch_count() + m.graph_launches - l0) // args.steps
            res[name].append(49 * args.steps / (e0.elapsed_time(e1) / 1e3))
            release(m)
    clocks = sampler.stop()
    per_step = {}
    for name, m in models.items():
        per_step[name] = profile(m, lr, img, args.steps, C)
        release(m)
    out = dict(
        gpu=dict(gpu, median_sm_clock_mhz=clocks.get('sm_mhz'), clock_reasons=clocks.get('reasons')),
        workload='Depth-Anything-vitl PatchFusion, 4K P49, cai_mode m2, process_num 9, synthetic weights',
        tiles_per_s={n: [round(x, 2) for x in v] for n, v in res.items()},
        median_tiles_per_s={n: round(statistics.median(v), 2) for n, v in res.items()},
        spread_tiles_per_s={n: round(max(v) - min(v), 2) for n, v in res.items()},
        launches_per_step=launches,
        per_step_ms=per_step,
        depth=depth)
    p = os.path.join(args.out, 'fp8_dpt_bench.json')
    with open(p, 'w') as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
