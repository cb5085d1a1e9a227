"""Runs the reference's own geometry helpers (`external/zoedepth/utils/geometry.py`: get_intrinsics, depth_to_points,
create_triangles) on seeded depth maps and writes tests/golden/geometry_case0.npz, which pins the numpy restatement in
tests/geometry_ref.py that the GPU tests of patchfusion_b200/geometry.py compare against.
python -m oracle.make_golden_geometry  (needs $PATCHFUSION_REFERENCE)

Cases: 7 x 9, 30 x 41 and 64 x 64 depth maps (fp32, uniform in [0.5, 20)), each with the identity pose and with a
seeded rotation R and translation t, and create_triangles without a mask and with a seeded 50 % vertex mask.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh         # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden', 'geometry_case0.npz')
SIZES = ((7, 9), (30, 41), (64, 64))


def rotation(rng):
    """Rodrigues rotation about a random axis by an angle in [0.2, 1.2) rad"""
    k = rng.normal(size=3)
    k /= np.linalg.norm(k)
    a = rng.uniform(0.2, 1.2)
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(a) * Kx + (1 - np.cos(a)) * Kx @ Kx


def main():
    rh._enter()
    from zoedepth.utils import geometry as g
    out = {}
    for i, (H, W) in enumerate(SIZES):
        rng = np.random.default_rng(i)
        tag = '%dx%d' % (H, W)
        depth = rng.uniform(0.5, 20.0, (1, H, W)).astype(np.float32)
        R, t = rotation(rng), rng.uniform(-3.0, 3.0, 3)
        mask = rng.random((H, W)) < 0.5
        out['depth_' + tag] = depth
        out['K_' + tag] = g.get_intrinsics(H, W)
        out['points_' + tag] = g.depth_to_points(depth)
        out['R_' + tag], out['t_' + tag] = R, t
        out['points_rt_' + tag] = g.depth_to_points(depth, R, t)
        out['mask_' + tag] = mask
        out['tri_' + tag] = g.create_triangles(H, W)
        out['tri_mask_' + tag] = g.create_triangles(H, W, mask)
        print('%s: %d triangles, %d kept by the mask' % (tag, len(out['tri_' + tag]), len(out['tri_mask_' + tag])))
    np.savez_compressed(OUT, **out)
    print('wrote', OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
