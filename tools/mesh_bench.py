"""Times the GPU depth-to-mesh passes of patchfusion_b200/geometry.py at 1080p, 4K and 8K, and the numpy
restatement of the reference's geometry.py (tests/geometry_ref.py) on one host thread for comparison.

    python tools/mesh_bench.py --out DIR

Phases, each timed with CUDA events over a warmed window of --iters calls:
  points     pf_depth_to_points with the image: depth + planar RGB in, points + colours out
  mask       pf_depth_edge_mask
  triangles  pf_mesh_quad_counts (counts + scan) and pf_mesh_triangles with that mask, into a buffer sized once
  ply        pf_ply_pack_vertices + pf_ply_pack_faces
Achieved GB/s uses the bytes each phase must move, computed from the shapes (neighbour re-reads counted once), against
the H100 SXM data sheet's 3.35 TB/s.  The card's name and power limit are read in the same run.  Writes DIR/mesh_bench.json.
"""
import os

for _v in ('OMP_NUM_THREADS', 'OPENBLAS_NUM_THREADS', 'MKL_NUM_THREADS'):
    os.environ[_v] = '1'                      # the host restatement runs on one thread, before numpy loads BLAS

import argparse
import json
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import numpy as np
import torch

import geometry_ref as gr
from patchfusion_b200 import geometry, ops

SIZES = {'1080p': (1080, 1920), '4K': (2160, 3840), '8K': (4320, 7680)}
HBM_TBPS = 3.35


def card():
    info = {'name': torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info['power_limit'], info['max_sm_clock'] = [s.strip() for s in out.split(',')]
    except Exception as e:                    # noqa: BLE001
        info['power_limit'] = 'unknown (%s)' % e
    return info


def timed(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def host_mem_gb():
    try:
        for line in open('/proc/meminfo'):
            if line.startswith('MemAvailable:'):
                return int(line.split()[1]) / 2 ** 20
    except OSError:
        pass
    return 0.0


def run_size(name, H, W, args, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    # a smooth surface with a few steps: the edge mask drops a few percent of the vertices, as on real depth
    y = torch.linspace(0, 1, H, device=dev)[:, None]
    x = torch.linspace(0, 1, W, device=dev)[None, :]
    depth = (5 + 3 * y + 2 * x + 4 * ((x > 0.5) & (y > 0.3)) + 0.01 * torch.rand(H, W, device=dev, generator=g))
    depth = depth[None].contiguous()
    image = torch.rand(1, 3, H, W, device=dev, generator=g)
    n, nq = H * W, (H - 1) * (W - 1)
    nb = ops.mesh_scan_blocks(H, W)
    inv_f = geometry._inv_f(W)
    points = torch.empty(n, 3, device=dev)
    colors = torch.empty(n, 3, dtype=torch.uint8, device=dev)
    mask = torch.empty(H, W, dtype=torch.bool, device=dev)
    flags = torch.empty(nq, dtype=torch.uint8, device=dev)
    offs = torch.empty(nb + 1, dtype=torch.int64, device=dev)
    ops.depth_edge_mask(depth, args.threshold, mask)
    ops.mesh_quad_counts(mask, H, W, flags, offs)
    nt = int(offs[nb].item())
    faces = torch.empty(nt, 3, dtype=torch.int32, device=dev)
    all_faces = torch.empty(2 * nq, 3, dtype=torch.int32, device=dev)
    vbytes = torch.empty(15 * n, dtype=torch.uint8, device=dev)
    fbytes = torch.empty(13 * nt, dtype=torch.uint8, device=dev)

    def tri():
        ops.mesh_quad_counts(mask, H, W, flags, offs)
        ops.mesh_triangles(flags, offs, H, W, faces)

    def ply():
        ops.ply_pack_vertices(points, colors, vbytes)
        ops.ply_pack_faces(faces, fbytes)

    phases = {
        'points': (lambda: ops.depth_to_points(depth, inv_f, None, image, points, colors), 4 * n + 12 * n + 12 * n + 3 * n),
        'mask': (lambda: ops.depth_edge_mask(depth, args.threshold, mask), 4 * n + n),
        'triangles': (tri, n + nq + 8 * nb + 2 * 8 * nb + nq + 8 * nb + 12 * nt),
        'triangles_unmasked': (lambda: ops.mesh_triangles(None, None, H, W, all_faces), 24 * nq),
        'ply': (ply, 15 * n + 15 * n + 12 * nt + 13 * nt),
    }
    res = {'size': name, 'H': H, 'W': W, 'vertices': n, 'triangles_kept': nt, 'triangles_all': 2 * nq,
           'scan_blocks': nb, 'phases': {}}
    for pname, (fn, nbytes) in phases.items():
        ms = timed(fn, args.iters, args.warmup)
        gbs = nbytes / ms / 1e6
        res['phases'][pname] = {'ms': ms, 'bytes': nbytes, 'GB/s': gbs, 'of_3.35TB/s': gbs / (HBM_TBPS * 1e3)}
    res['gpu_mesh_ms'] = sum(res['phases'][p]['ms'] for p in ('points', 'mask', 'triangles'))
    # the numpy restatement of geometry.py on the same depth: points, the edge mask and the masked triangles
    need_gb = 200e-9 * n                     # peak host memory of the restatement, measured loosely: ~200 bytes / pixel
    if args.no_host or host_mem_gb() < 2 * need_gb:
        res['host_numpy_s'] = None
        res['host_note'] = 'not measured (%s)' % ('--no-host' if args.no_host else
                                                  'needs ~%.0f GB of host memory, %.0f GB available' %
                                                  (need_gb, host_mem_gb()))
    else:
        d = depth.cpu().numpy()
        t0 = time.perf_counter()
        gr.depth_to_points(d)
        m = gr.edge_mask(d, args.threshold)
        gr.create_triangles(H, W, m)
        res['host_numpy_s'] = time.perf_counter() - t0
        res['host_note'] = 'numpy %s, 1 thread' % np.__version__
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--sizes', nargs='+', default=list(SIZES), choices=list(SIZES))
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--threshold', type=float, default=0.05)
    ap.add_argument('--no-host', action='store_true')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('mesh_bench: no GPU visible; these timings only mean something on the device')
    dev = torch.device('cuda:0')
    os.makedirs(args.out, exist_ok=True)
    out = {'card': card(), 'hbm_datasheet_TB/s': HBM_TBPS, 'iters': args.iters, 'results': []}
    print('card: %s, power limit %s' % (out['card']['name'], out['card'].get('power_limit')))
    for name in args.sizes:
        r = run_size(name, *SIZES[name], args, dev)
        out['results'].append(r)
        print('%-5s %dx%d: %d vertices, %d of %d triangles kept, %d scan blocks' %
              (name, r['H'], r['W'], r['vertices'], r['triangles_kept'], r['triangles_all'], r['scan_blocks']))
        for p, v in r['phases'].items():
            print('    %-19s %8.3f ms  %7.1f GB/s  (%.0f %% of 3.35 TB/s)' % (p, v['ms'], v['GB/s'],
                                                                           100 * v['of_3.35TB/s']))
        host = '%.2f s' % r['host_numpy_s'] if r['host_numpy_s'] is not None else '-'
        print('    GPU points + mask + triangles %.3f ms; host %s (%s)' % (r['gpu_mesh_ms'], host, r['host_note']))
    path = os.path.join(args.out, 'mesh_bench.json')
    with open(path, 'w') as f:
        json.dump(out, f, indent=1)
    print('wrote', path)


if __name__ == '__main__':
    main()
