"""Batched inference throughput of PatchFusion (Depth-Anything-vitl, synthetic weights): one image per forward against
one forward over B images, alternated in the same process.

    python tools/batch_bench.py --out DIR [--batches 2,4,8] [--repeats 3] [--warmup 1] [--all-gpus]

configurations  4K P49        2160x3840, 4x4 split, m2 (49 tiles per image), process_num 9
                1080p m1      1080x1920, 2x2 split, m1 (4 tiles per image), process_num 9
                1080p m2      1080x1920, 2x2 split, m2 (9 tiles per image), process_num 9

For every configuration and B, one timed window runs the same B images either as B single-image forwards or as one
batched forward; the two kinds of window alternate, `repeats` of each after `warmup` of each (packing, graph capture),
and every window ends in a device synchronise.  images/s and tiles/s are medians with their spread.
--all-gpus: when more than one GPU is visible, the same is measured tile-sharded over all of them (torch.distributed.run
with NCCL, rank 0 reports); on one GPU that part is reported as not measured.  The card's name, power limit and max SM
clock are read with nvidia-smi (read-only query) in the same run.  Writes DIR/batch_bench[_W<n>].json and prints it.
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

CONFIGS = [('4K_P49_m2', (2160, 3840), (4, 4), 'm2', 9, 49),
           ('1080p_2x2_m1', (1080, 1920), (2, 2), 'm1', 9, 4),
           ('1080p_2x2_m2', (1080, 1920), (2, 2), 'm2', 9, 9)]


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        name, power, clock = [s.strip() for s in out[0].split(',')]
        return dict(name=name, power_limit=power, max_sm_clock=clock, visible_gpus=torch.cuda.device_count())
    except Exception as e:                              # the timings stand; the card is then reported unknown
        return dict(error=repr(e))


def _stats(rates):
    return dict(median=statistics.median(rates), min=min(rates), max=max(rates), repeats=len(rates))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--batches', default='2,4,8')
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=1)
    ap.add_argument('--configs', default=','.join(c[0] for c in CONFIGS))
    ap.add_argument('--all-gpus', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('batch_bench: no CUDA device (this measures the H100 path only)')
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    if args.all_gpus and world == 1:
        n = torch.cuda.device_count()
        res = run(args, None, None)
        if n < 2:
            res['sharded'] = 'not measured: %d GPU visible' % n
            print('sharded over all GPUs: not measured (%d GPU visible)' % n, flush=True)
        else:
            cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', str(n),
                   '--master-addr', '127.0.0.1', '--master-port', '29651', os.path.abspath(__file__),
                   '--out', args.out, '--batches', args.batches, '--repeats', str(args.repeats),
                   '--warmup', str(args.warmup), '--configs', args.configs]
            rc = subprocess.run(cmd).returncode
            res['sharded'] = 'batch_bench_W%d.json' % n if rc == 0 else 'failed (exit %d)' % rc
        _write(args.out, 'batch_bench.json', res)
        return
    group = None
    if world > 1:
        import torch.distributed as dist
        local = int(os.environ['LOCAL_RANK'])
        torch.cuda.set_device(local)
        dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    res = run(args, (rank, world) if world > 1 else None, group)
    if rank == 0:
        _write(args.out, 'batch_bench.json' if world == 1 else 'batch_bench_W%d.json' % world, res)
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()


def _write(out, name, res):
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, name), 'w') as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res), flush=True)


def run(args, shard, group):
    from patchfusion_b200.configs import depth_anything_patchfusion
    from patchfusion_b200.model import PatchFusion
    dev = torch.device('cuda', torch.cuda.current_device())
    cfg = depth_anything_patchfusion('vitl')
    model = PatchFusion(cfg).init_synthetic_weights(0).to(dev).eval()
    world = 1 if shard is None else shard[1]
    talk = shard is None or shard[0] == 0
    res = dict(metric='PatchFusion vitl: one image per forward vs B images per forward', world=world, card=card(),
               shard_coarse=model.shard_coarse if world > 1 else None, configs={})
    batches = [int(b) for b in args.batches.split(',')]
    g = torch.Generator().manual_seed(0)
    for name, shape, split, mode, pn, tiles in CONFIGS:
        if name not in args.configs.split(','):
            continue
        tcfg = {'image_raw_shape': list(shape), 'patch_split_num': list(split)}
        imgs = torch.rand(max(batches), 3, *shape, generator=g).to(dev)
        lrs = model.make_lr(imgs)
        entry = {}
        for B in batches:
            def single():
                for b in range(B):
                    model(mode='infer', image_lr=lrs[b:b + 1], image_hr=imgs[b:b + 1], tile_cfg=tcfg, cai_mode=mode,
                          process_num=pn, shard=shard, group=group)

            def batched():
                model(mode='infer', image_lr=lrs[:B], image_hr=imgs[:B], tile_cfg=tcfg, cai_mode=mode,
                      process_num=pn, shard=shard, group=group)
            rates = {'single': [], 'batched': []}
            for it in range(args.warmup + args.repeats):
                for kind, fn in (('single', single), ('batched', batched)):
                    random.seed(0)
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    fn()
                    torch.cuda.synchronize()
                    if it >= args.warmup:
                        rates[kind].append(B / (time.perf_counter() - t0))
            e = {k: dict(images_per_s=_stats(v), tiles_per_s=statistics.median(v) * tiles) for k, v in rates.items()}
            e['speedup'] = e['batched']['images_per_s']['median'] / e['single']['images_per_s']['median']
            entry['B%d' % B] = e
            if talk:
                print('%s world %d B=%d: one image per forward %.3f images/s (%.1f tiles/s), batched %.3f images/s '
                      '(%.1f tiles/s), x%.3f' % (name, world, B, e['single']['images_per_s']['median'],
                                                 e['single']['tiles_per_s'], e['batched']['images_per_s']['median'],
                                                 e['batched']['tiles_per_s'], e['speedup']), flush=True)
        res['configs'][name] = dict(image_raw_shape=shape, patch_split_num=split, cai_mode=mode, process_num=pn,
                                    tiles_per_image=tiles, **entry)
        del imgs, lrs
        model.invalidate()
        torch.cuda.empty_cache()
    return res


if __name__ == '__main__':
    main()
