"""Throughput of BaselinePretrain (the paper's coarse-only and fine-only baselines), Depth-Anything-vitl, synthetic
weights.

    python tools/baseline_bench.py --out DIR [--repeats 5] [--warmup 2]

coarse target   images/s at 392x518 for B in {1, 8, 32}
fine target     tiles/s and 4K images/s at P49 (m2, process_num 9) and at r128 (49 + 128 x 9 random tiles)

Each figure: warm-up calls first (packing, graph capture), then `repeats` timed windows, each closed by a device
synchronise; the median and the spread are reported.  `tflops` is rate x 970.1 GF per 392x518 branch image (SURVEY.md
§6): a whole-program rate, not a kernel's share of peak.  The card's name, power limit and max SM clock are read
with nvidia-smi (read-only query) in the same run.  Writes DIR/baseline_bench.json and prints it.
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

GF_BRANCH = 970.1e9          # one vitl branch forward at 392x518 (SURVEY.md §6)


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [s.strip() for s in out.split(',')]
        return dict(name=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:                              # the timings stand; the card is then reported unknown
        return dict(error=repr(e))


def timed(fn, repeats, warmup, units):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    rates = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        rates.append(units / (time.perf_counter() - t0))
    return dict(median=statistics.median(rates), min=min(rates), max=max(rates), repeats=repeats)


def model_cfg(target):
    import copy
    from patchfusion_b200.configs import _BRANCH
    br = dict(copy.deepcopy(_BRANCH), midas_model_type='vitl')
    cfg = dict(min_depth=1e-3, max_depth=80, target=target, coarse_branch=br, fine_branch=copy.deepcopy(br),
               sigloss=dict(type='SILogLoss'))
    if target == 'fine':
        cfg['patch_process_shape'] = (392, 518)
    return cfg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--repeats', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--batches', default='1,8,32')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('baseline_bench: no CUDA device (this measures the H100 path only)')
    from patchfusion_b200.baseline import BaselinePretrain
    dev = torch.device('cuda:0')
    res = dict(metric='BaselinePretrain vitl throughput', gf_per_branch_image=GF_BRANCH / 1e9, card=card(),
               coarse={}, fine={})
    g = torch.Generator().manual_seed(0)

    coarse = BaselinePretrain(**model_cfg('coarse')).init_synthetic_weights(0).to(dev).eval()
    for B in [int(b) for b in args.batches.split(',')]:
        lr = torch.rand(B, 3, 392, 518, generator=g).to(dev)
        r = timed(lambda: coarse(mode='infer', image_lr=lr, image_hr=None), args.repeats, args.warmup, B)
        r['tflops'] = r['median'] * GF_BRANCH / 1e12
        res['coarse']['B%d' % B] = dict(images_per_s=r)
        print('coarse B=%d: %.1f images/s (%.0f TFLOP/s whole-program)' % (B, r['median'], r['tflops']), flush=True)
    del coarse, lr
    torch.cuda.empty_cache()

    fine = BaselinePretrain(**model_cfg('fine')).init_synthetic_weights(0).to(dev).eval()
    img = torch.rand(1, 3, 2160, 3840, generator=g).to(dev)
    for name, mode, pn, tiles in (('P49_m2', 'm2', 9, 49), ('r128', 'r128', 9, 49 + 128 * 9)):
        def step():
            random.seed(0)
            fine(mode='infer', image_lr=None, image_hr=img, cai_mode=mode, process_num=pn)
        r = timed(step, args.repeats, args.warmup, 1)
        res['fine'][name] = dict(cai_mode=mode, process_num=pn, tiles_per_image=tiles, images_per_s=r,
                                 tiles_per_s=r['median'] * tiles, tflops=r['median'] * tiles * GF_BRANCH / 1e12)
        print('fine %s: %.3f images/s, %.1f tiles/s (%.0f TFLOP/s whole-program)' %
              (name, r['median'], r['median'] * tiles, r['median'] * tiles * GF_BRANCH / 1e12), flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'baseline_bench.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
