"""Calibrated FP8 BaselinePretrain measurement: the arms bf16, ViT FP8 (branch_vit_precision 'fp8_static') and ViT + DPT
FP8 (branch_vit_precision and branch_dpt_precision 'fp8_static') of Depth-Anything-vitl with synthetic weights on

    coarse target   images/s at 392x518, B = 1, 8 and 32
    fine target     tiles/s at 4K P49 (cai_mode m2, process_num 9)

    python tools/fp8_baseline_bench.py --out DIR [--windows 3] [--calib-images 2]

The FP8 models are calibrated first (BaselinePretrain.calibrate_fp8) on seeded random images that are not the timed
ones: the coarse models on --calib-images 392x518 images in one batch, the fine models on --calib-images 4K images in
m2.  Per workload the arms alternate in timed windows (two untimed steps before each window rebuild what the previous
arm's release dropped; each window ends in a device synchronise) and the median over --windows windows is reported
with the spread (max - min).  Writes DIR/fp8_baseline_bench.json and prints it:
  * gpu: card name and power limit (nvidia-smi, in the same process), median SM clock over the timed windows;
  * per workload and arm: the rate of each window, its median and spread, and the speed-up over bf16;
  * depth: max-abs / mean-abs difference of each FP8 arm from bf16 on the timed input, and bf16's range.
"""
import argparse
import copy
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
from fp8_vit_bench import release   # noqa: E402

ARMS = {'bf16': {}, 'vit_fp8': dict(branch_vit_precision='fp8_static'),
        'vit_dpt_fp8': dict(branch_vit_precision='fp8_static', branch_dpt_precision='fp8_static')}
# steps per timed window: each window is several hundred ms of GPU work
COARSE_STEPS = {1: 96, 8: 16, 32: 4}
FINE_STEPS = 3


def model_cfg(target, **kw):
    from patchfusion_b200.configs import _BRANCH
    br = dict(copy.deepcopy(_BRANCH), midas_model_type='vitl')
    cfg = dict(min_depth=1e-3, max_depth=80, target=target, coarse_branch=br, fine_branch=copy.deepcopy(br),
               sigloss=dict(type='SILogLoss'), **kw)
    if target == 'fine':
        cfg['patch_process_shape'] = (392, 518)
    return cfg


def compare(arms, step, units, steps, windows):
    """{arm: rates of its windows}, {arm: depth of one step (cloned)}: the arms alternate, window by window"""
    outs, rates = {}, {n: [] for n in arms}
    for name, m in arms.items():
        for _ in range(3):
            outs[name] = step(m).clone()
        release(m)
    for _ in range(windows):
        for name, m in arms.items():
            for _ in range(2):
                step(m)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                step(m)
            e1.record()
            torch.cuda.synchronize()
            rates[name].append(units * steps / (e0.elapsed_time(e1) / 1e3))
            release(m)
    return rates, outs


def summary(rates, outs, unit):
    med = {n: statistics.median(v) for n, v in rates.items()}
    out = {n: {unit: [round(x, 2) for x in v], 'median': round(med[n], 2), 'spread': round(max(v) - min(v), 2),
               'vs_bf16': round(med[n] / med['bf16'], 4)} for n, v in rates.items()}
    for n in outs:
        if n != 'bf16':
            d = (outs[n] - outs['bf16']).abs()
            out[n]['depth_vs_bf16'] = dict(max_abs=d.max().item(), mean_abs=d.mean().item())
    out['bf16']['depth_range'] = [outs['bf16'].min().item(), outs['bf16'].max().item()]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--windows', type=int, default=3)
    ap.add_argument('--calib-images', type=int, default=2)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('fp8_baseline_bench: no CUDA device (the measurement runs on the GPU only)')
    os.makedirs(args.out, exist_ok=True)
    import bench
    from patchfusion_b200.baseline import BaselinePretrain
    gpu = gpu_info()
    dev = torch.device('cuda')
    sampler = bench.ClockSampler(torch.cuda.current_device())
    res = {}

    def build(target):
        arms = {}
        for name, kw in ARMS.items():
            arms[name] = BaselinePretrain(**model_cfg(target, **kw)).init_synthetic_weights(0).to(dev).eval()
        return arms

    arms = build('coarse')
    cal = torch.rand(args.calib_images, 3, 392, 518, generator=torch.Generator().manual_seed(1234)).to(dev)
    for name, m in arms.items():
        if name != 'bf16':
            m.calibrate_fp8(cal, None)
            release(m)
    for B in COARSE_STEPS:
        lr = torch.rand(B, 3, 392, 518, generator=torch.Generator().manual_seed(7 + B)).to(dev)
        rates, outs = compare(arms, lambda m: m(mode='infer', image_lr=lr, image_hr=None)[0], B, COARSE_STEPS[B],
                              args.windows)
        res['coarse_392x518_B%d' % B] = summary(rates, outs, 'images_per_s')
        print(json.dumps({'coarse B=%d' % B: res['coarse_392x518_B%d' % B]}), flush=True)
    del arms, outs
    torch.cuda.empty_cache()

    arms = build('fine')
    cal = torch.rand(args.calib_images, 3, 2160, 3840, generator=torch.Generator().manual_seed(1234)).to(dev)
    for name, m in arms.items():
        if name != 'bf16':
            random.seed(0)
            m.calibrate_fp8(None, cal, cai_mode='m2', process_num=9)
            release(m)
    del cal
    img = torch.rand(1, 3, 2160, 3840, generator=torch.Generator().manual_seed(7)).to(dev)
    rates, outs = compare(arms, lambda m: m(mode='infer', image_lr=None, image_hr=img, cai_mode='m2',
                                            process_num=9)[0], 49, FINE_STEPS, args.windows)
    res['fine_4k_P49_m2_pn9'] = summary(rates, outs, 'tiles_per_s')
    clocks = sampler.stop()
    out = dict(gpu=dict(gpu, median_sm_clock_mhz=clocks.get('sm_mhz'), clock_reasons=clocks.get('reasons')),
               workload='BaselinePretrain Depth-Anything-vitl, synthetic weights: coarse target 392x518 images/s, '
                        'fine target 4K P49 (m2, process_num 9) tiles/s',
               windows=args.windows, **res)
    with open(os.path.join(args.out, 'fp8_baseline_bench.json'), 'w') as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
