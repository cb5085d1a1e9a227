"""FP8 U-Net measurement: fusion_precision 'bf16' against 'fp8' on the vitl 4K P49 workload (cai_mode m2, process_num 9).

    python tools/fp8_bench.py --out DIR [--steps 3] [--windows 3]

Writes DIR/fp8_bench.json and prints it:
  * gpu: card name, power limit, median SM clock over the timed windows (nvidia-smi);
  * per_conv: every covered 3x3 conv shape, by launch label (summed over its launches in a step), from the library's
    per-launch CUDA events over `--steps` profiled steps of each model: bf16 conv ms and TFLOP/s against the FP8 conv,
    its own amax and quantize launches, the net gain, and the quantize passes' achieved bandwidth (bf16 sources read
    twice + the e4m3 map written);
  * workload: tiles/s of each model in alternated timed windows (CUDA events), launches per step;
  * depth: max-abs and mean-abs difference of the FP8 model's depth from the bf16 model's on the same image.
Weights are the seeded synthetic ones (no trained checkpoints offline): the depth difference is the quantization cost
on those weights, not an accuracy figure.
"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        out = subprocess.check_output(['nvidia-smi', '-i', str(torch.cuda.current_device()),
                                       '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                                      text=True).strip()
        name, plim, smax = [s.strip() for s in out.split(',')]
        return dict(name=name, power_limit=plim, sm_max_clock=smax)
    except Exception as e:     # the card name from torch at least
        return dict(name=torch.cuda.get_device_name(), power_limit='unknown (%s)' % e)


def profile_convs(model, lr, img, steps):
    """label -> list of per-step ms summed over the launches with that label (one micro-batch's covered convs)"""
    from patchfusion_b200 import lib
    per = {}
    for _ in range(steps):
        prof = lib.Profiler()
        lib.PROFILER = prof
        try:
            prof.start()
            model(mode='infer', image_lr=lr, image_hr=img, cai_mode='m2', process_num=9)
            recs = prof.stop()
        finally:
            lib.PROFILER = None
        # an FP8 conv is launched right after its amax and quantize launches: they are booked to its label
        step, pending = {}, []
        for name, label, flops, ms in recs:
            if name in ('quant_amax_kernel', 'quant_write_kernel'):
                pending.append((name, label, ms))
                continue
            if name not in ('pf_conv3_halo_kernel', 'pf_conv3_halo_e4m3_kernel'):
                continue
            d = step.setdefault((name, label), dict(ms=0.0, flops=0.0, launches=0, amax_ms=0.0, quant_ms=0.0,
                                                    quant_bytes=0.0))
            d['ms'] += ms
            d['flops'] += flops
            d['launches'] += 1
            if name == 'pf_conv3_halo_e4m3_kernel':
                assert [p_[0] for p_ in pending] == ['quant_amax_kernel', 'quant_write_kernel'], pending
                m_ = re.search(r'rows(\d+) K\d+x(\d+)', label)
                kq = re.search(r' K(\d+)$', pending[1][1])
                rows, k8 = int(m_.group(1)), int(m_.group(2))
                # amax reads the bf16 sources; quantize reads them again and writes one byte per e4m3 map channel
                d['amax_ms'] += pending[0][2]
                d['quant_ms'] += pending[1][2]
                d['quant_bytes'] += 2 * rows * k8 * 2 + rows * int(kq.group(1))
            pending = []
        for k, v in step.items():
            per.setdefault(k, []).append(v)
    return {k: dict({f: statistics.median(x[f] for x in v) for f in ('ms', 'amax_ms', 'quant_ms')},
                    flops=v[0]['flops'], launches=v[0]['launches'], quant_bytes=v[0]['quant_bytes'])
            for k, v in per.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--steps', type=int, default=3)
    ap.add_argument('--windows', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('fp8_bench: no CUDA device (the measurement runs on the GPU only)')
    os.makedirs(args.out, exist_ok=True)
    import bench
    from patchfusion_b200 import lib
    from patchfusion_b200.model import PatchFusion
    dev = torch.device('cuda')
    cfg, sd = bench.build_inputs('vitl')
    models = {}
    for prec in ('bf16', 'fp8'):
        m = PatchFusion(dict(cfg, fusion_precision=prec))
        m.load_state_dict(sd, strict=True)
        models[prec] = m.to(dev).eval()
    img = torch.rand(1, 3, 2160, 3840, generator=torch.Generator().manual_seed(7)).to(dev)
    lr = models['bf16'].make_lr(img)
    n_tiles = None

    def step(m):
        return m(mode='infer', image_lr=lr, image_hr=img, cai_mode='m2', process_num=9)[0]

    outs = {}
    for prec, m in models.items():
        for _ in range(3):
            outs[prec] = step(m).clone()
    torch.cuda.synchronize()
    d = (outs['fp8'] - outs['bf16']).abs()
    depth = dict(max_abs=d.max().item(), mean_abs=d.mean().item(),
                 bf16_range=[outs['bf16'].min().item(), outs['bf16'].max().item()])

    sampler = bench.ClockSampler(torch.cuda.current_device())
    res = {p: [] for p in models}
    launches = {}
    for w in range(args.windows):
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
            if n_tiles is None:
                n_tiles = 49
            res[prec].append(n_tiles * args.steps / (e0.elapsed_time(e1) / 1e3))
    clocks = sampler.stop()

    per = {p: profile_convs(m, lr, img, args.steps) for p, m in models.items()}
    # pair each bf16 conv with the FP8 conv of the same shape (labels differ only in the kernel tag)
    convs = []
    for (name, label), v in sorted(per['bf16'].items(), key=lambda kv: -kv[1]['ms']):
        if name != 'pf_conv3_halo_kernel':
            continue
        k8 = ('pf_conv3_halo_e4m3_kernel', label.replace('conv3x3 ', 'conv3x3_e4m3 ', 1))
        if k8 not in per['fp8']:
            continue          # not a covered conv (fusion_conv_list, the branches' convs)
        f8 = per['fp8'][k8]
        m_ = re.search(r'rows(\d+) K(\d+)x(\d+)', label)
        kc = int(m_.group(3)) if m_ else 0
        q_ms = f8['amax_ms'] + f8['quant_ms']
        convs.append(dict(label=label, launches=v['launches'], bf16_ms=v['ms'], fp8_conv_ms=f8['ms'],
                          fp8_amax_ms=f8['amax_ms'], fp8_quantize_ms=f8['quant_ms'], fp8_total_ms=f8['ms'] + q_ms,
                          net_gain_ms=v['ms'] - f8['ms'] - q_ms,
                          bf16_tflops=v['flops'] / (v['ms'] * 1e9) if v['ms'] else None,
                          fp8_tflops=f8['flops'] / (f8['ms'] * 1e9) if f8['ms'] else None,
                          quantize_gbs=f8['quant_bytes'] / (q_ms * 1e6) if q_ms else None, k_true=kc))
    q_ms = sum(c['fp8_amax_ms'] + c['fp8_quantize_ms'] for c in convs)
    q_bytes = sum(per['fp8'][('pf_conv3_halo_e4m3_kernel', c['label'].replace('conv3x3 ', 'conv3x3_e4m3 ', 1))]
                  ['quant_bytes'] for c in convs)
    out = dict(
        gpu=dict(gpu_info(), median_sm_clock_mhz=clocks.get('sm_mhz'), clock_reasons=clocks.get('reasons')),
        workload='Depth-Anything-vitl PatchFusion, 4K P49, cai_mode m2, process_num 9, synthetic weights',
        workload_tiles_per_s={p: [round(x, 2) for x in v] for p, v in res.items()},
        workload_median_tiles_per_s={p: round(statistics.median(v), 2) for p, v in res.items()},
        launches_per_step=launches,
        per_conv=convs,
        per_step_ms=dict(bf16_covered_convs=sum(c['bf16_ms'] for c in convs),
                         fp8_covered_convs=sum(c['fp8_conv_ms'] for c in convs), fp8_quantize=q_ms,
                         fp8_quantize_gbs=q_bytes / (q_ms * 1e6) if q_ms else None),
        depth_fp8_vs_bf16=depth)
    p = os.path.join(args.out, 'fp8_bench.json')
    with open(p, 'w') as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
