"""Mixed-geometry batched inference throughput of PatchFusion (Depth-Anything-vitl, synthetic weights) on one GPU: a
stream that alternates a 4K image (2160x3840, 4x4 split, m2: 49 tiles) and a 1080p image (1080x1920, 2x2 split, m1:
4 tiles), process_num 9, run as one image per forward against one mixed forward over B images, alternated in the
same process.

    python tools/mixed_batch_bench.py --out DIR [--batches 2,4,8] [--repeats 3] [--warmup 1]

For every B, one timed window runs the first B images of the stream either as B single-image forwards or as one mixed
forward (image_hr, tile_cfg and cai_mode as lists); the two kinds of window alternate, `repeats` of each after `warmup`
of each (packing, graph capture), and every window ends in a device synchronise.  images/s and tiles/s are medians
with their spread.  The card's name, power limit and max SM clock are read with nvidia-smi (read-only query) in the
same run.  Writes DIR/mixed_batch_bench.json and prints it.
"""
import argparse
import json
import os
import random
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

from tools.batch_bench import _stats, card  # noqa: E402

# (name, image_raw_shape, patch_split_num, cai_mode, tiles per image): the two arms of the stream, alternated
STREAM = [('4K_P49_m2', (2160, 3840), (4, 4), 'm2', 49), ('1080p_2x2_m1', (1080, 1920), (2, 2), 'm1', 4)]
PROCESS_NUM = 9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--batches', default='2,4,8')
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('mixed_batch_bench: no CUDA device (this measures the H100 path only)')
    from patchfusion_b200.configs import depth_anything_patchfusion
    from patchfusion_b200.model import PatchFusion
    dev = torch.device('cuda', torch.cuda.current_device())
    model = PatchFusion(depth_anything_patchfusion('vitl')).init_synthetic_weights(0).to(dev).eval()
    batches = [int(b) for b in args.batches.split(',')]
    g = torch.Generator().manual_seed(0)
    arms = [STREAM[i % len(STREAM)] for i in range(max(batches))]
    imgs = [torch.rand(1, 3, *a[1], generator=g).to(dev) for a in arms]
    cfgs = [{'image_raw_shape': list(a[1]), 'patch_split_num': list(a[2])} for a in arms]
    modes = [a[3] for a in arms]
    lrs = model.make_lr(imgs)
    res = dict(metric='PatchFusion vitl, mixed stream: one image per forward vs B images per forward', card=card(),
               stream=[dict(name=n, image_raw_shape=s, patch_split_num=p, cai_mode=m, tiles_per_image=t)
                       for n, s, p, m, t in STREAM], process_num=PROCESS_NUM, batches={})
    for B in batches:
        tiles = sum(a[4] for a in arms[:B])

        def single():
            for b in range(B):
                model(mode='infer', image_lr=lrs[b:b + 1], image_hr=imgs[b], tile_cfg=cfgs[b], cai_mode=modes[b],
                      process_num=PROCESS_NUM)

        def mixed():
            model(mode='infer', image_lr=lrs[:B], image_hr=imgs[:B], tile_cfg=cfgs[:B], cai_mode=modes[:B],
                  process_num=PROCESS_NUM)
        rates = {'single': [], 'mixed': []}
        for it in range(args.warmup + args.repeats):
            for kind, fn in (('single', single), ('mixed', mixed)):
                random.seed(0)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn()
                torch.cuda.synchronize()
                if it >= args.warmup:
                    rates[kind].append(B / (time.perf_counter() - t0))
        e = {k: dict(images_per_s=_stats(v), tiles_per_s=statistics.median(v) * tiles / B) for k, v in rates.items()}
        e['speedup'] = e['mixed']['images_per_s']['median'] / e['single']['images_per_s']['median']
        e['images'] = [a[0] for a in arms[:B]]
        res['batches']['B%d' % B] = e
        print('mixed stream B=%d: one image per forward %.3f images/s (%.1f tiles/s), mixed %.3f images/s '
              '(%.1f tiles/s), x%.3f' % (B, e['single']['images_per_s']['median'], e['single']['tiles_per_s'],
                                         e['mixed']['images_per_s']['median'], e['mixed']['tiles_per_s'],
                                         e['speedup']), flush=True)
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, 'mixed_batch_bench.json'), 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
