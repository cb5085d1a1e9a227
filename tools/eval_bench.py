"""python tools/eval_bench.py --out DIR [--frames 16] [--windows 2] : is host-side data preparation a bound on the
U4K evaluation loop?

Writes a synthetic U4K tree (raw 2160x3840 frames, fp32 disparities) and runs the evaluation loop (PreparedSamples ->
Tester.run, vitl synthetic weights, 4K, tiles 4x4) for m1 and m2 with two preparations, in alternated windows:
  gpu   raw bytes read on the reader thread into the pinned ring, copied as read, pf_ingest_raw_u8 + pf_gt_prepare on
        the device;
  host  the reference's preparation on the reader thread (numpy disparity -> depth, get_boundaries, float32 / 255)
        and fp32 copies of image, depth and boundary.
Reports images/s, host ms per image on the reader thread (reading the files plus, for `host`, the numpy preparation:
the same scope on both paths) and H2D bytes per image, on one GPU and, through torchrun, on all visible GPUs (images
sharded as tools/test.py --launcher pytorch does).  Writes
DIR/eval_bench.json with the card name and power limit."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from patchfusion_b200 import datasets as D  # noqa: E402


class HostPrepared:
    """The dataset with the reference's host preparation done in __getitem__ (on the reader thread)."""

    def __init__(self, ds):
        self.ds, self.prep_ms, self.h2d = ds, [], []

    def __len__(self):
        return len(self.ds)

    def __getitem__(self, i):
        t = time.perf_counter()
        s = self.ds[i]
        depth, boundary = D.host_ground_truth(s['gt'], s['gt_kind'], s['factor'], s['doffs'])
        image = np.ascontiguousarray(D.host_image(s['image']).transpose(2, 0, 1))[None]
        self.prep_ms.append((time.perf_counter() - t) * 1e3)
        out = dict(image=image, gt=depth[None, None], boundary=boundary[None, None],
                   img_file_basename=s['img_file_basename'])
        self.h2d.append(image.nbytes + depth.nbytes + boundary.nbytes)
        return out

    @staticmethod
    def prepare(s, device):
        return dict(image_hr=s['image'].to(device, non_blocking=True), depth_gt=s['gt'].to(device, non_blocking=True),
                    boundary=s['boundary'].to(device, non_blocking=True), img_file_basename=s['img_file_basename'])

    def reset(self):
        self.prep_ms, self.h2d = [], []


class GpuPrepared(HostPrepared):
    def __getitem__(self, i):
        t = time.perf_counter()
        s = self.ds[i]
        s = dict(s, gt=np.ascontiguousarray(s['gt']))           # the .npy is read from its memory map here
        self.prep_ms.append((time.perf_counter() - t) * 1e3)
        self.h2d.append(s['image'].nbytes + s['gt'].nbytes)
        return s

    @staticmethod
    def prepare(s, device):
        return D.prepare(s, device)


def run_window(tester, wrapped, indices, dev, mode, world):
    wrapped.reset()
    if world > 1:
        torch.distributed.barrier()
    torch.cuda.synchronize()
    t = time.perf_counter()
    tester.run(D.PreparedSamples(wrapped, indices, dev, num_workers=2), cai_mode=mode, process_num=4,
               image_raw_shape=(2160, 3840), patch_split_num=(4, 4))
    torch.cuda.synchronize()
    if world > 1:
        torch.distributed.barrier()
    wall = time.perf_counter() - t
    return wall, float(np.mean(wrapped.prep_ms)), float(np.mean(wrapped.h2d))


def bench(root, rank, world, dev, windows):
    from patchfusion_b200.configs import depth_anything_patchfusion
    from patchfusion_b200.model import PatchFusion
    from patchfusion_b200.tester import Tester
    split = os.path.join(root, 'splits', 'val.txt')
    ds = D.UnrealStereo4kDataset('infer', root, split, {}, 1e-3, 80, resize_mode='depth-anything')
    indices = list(range(rank, len(ds), world))
    model = PatchFusion(depth_anything_patchfusion('vitl')).init_synthetic_weights(0).to(dev).eval()
    tester = Tester(model, min_depth=1e-3, max_depth=80)
    paths = {'gpu': GpuPrepared(ds), 'host': HostPrepared(ds)}
    out = {}
    for mode in ('m1', 'm2'):
        for name, w in paths.items():                               # warm-up: every shape of the timed windows
            run_window(tester, w, indices[:1], dev, mode, world)
        rec = {k: [] for k in paths}
        for _ in range(windows):
            for name in ('gpu', 'host') if _ % 2 == 0 else ('host', 'gpu'):
                rec[name].append(run_window(tester, paths[name], indices, dev, mode, world))
        out[mode] = {k: dict(images_per_s=[len(ds) / r[0] for r in v], host_ms_per_image=[r[1] for r in v],
                             h2d_bytes_per_image=v[0][2]) for k, v in rec.items()}
    return out


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def main():
    p = argparse.ArgumentParser()
    p.add_argument('--out', required=True)
    p.add_argument('--frames', type=int, default=16)
    p.add_argument('--windows', type=int, default=2)
    p.add_argument('--worker', default=None, help='(internal) tree root, under torchrun')
    args = p.parse_args()
    os.makedirs(args.out, exist_ok=True)
    if args.worker:
        import torch.distributed as dist
        local = int(os.environ['LOCAL_RANK'])
        dev = torch.device('cuda', local)
        torch.cuda.set_device(dev)
        dist.init_process_group('nccl', device_id=dev)
        res = bench(args.worker, dist.get_rank(), dist.get_world_size(), dev, args.windows)
        if dist.get_rank() == 0:
            json.dump(res, open(os.path.join(args.out, 'eval_bench_all.json'), 'w'), indent=1)
        dist.destroy_process_group()
        return
    from patchfusion_b200 import eval_tree
    assert torch.cuda.is_available(), 'eval_bench measures on the GPU'
    with tempfile.TemporaryDirectory(prefix='pf_eval_bench_') as tmp:
        eval_tree.write_u4k_tree(tmp, args.frames, seed=0)
        report = dict(card=card(), frames=args.frames, encoder='vitl', tiles='4x4', windows=args.windows)
        report['one_gpu'] = bench(tmp, 0, 1, torch.device('cuda', 0), args.windows)
        print(json.dumps(report['one_gpu']), flush=True)
        n = torch.cuda.device_count()
        if n > 1:
            subprocess.check_call(['torchrun', '--standalone', '--nproc-per-node', str(n), os.path.abspath(__file__),
                                   '--out', args.out, '--windows', str(args.windows), '--worker', tmp])
            report['all_gpus'] = dict(gpus=n, **json.load(open(os.path.join(args.out, 'eval_bench_all.json'))))
    json.dump(report, open(os.path.join(args.out, 'eval_bench.json'), 'w'), indent=1)
    print(json.dumps(report, indent=1))


if __name__ == '__main__':
    main()
