"""Host side of patchfusion_b200/geometry.py (no GPU): the numpy restatement in tests/geometry_ref.py against the
reference's own geometry.py outputs (tests/golden/geometry_case0.npz, oracle/make_golden_geometry.py), the PLY writer
through a numpy reader, and the argument checks that must raise before anything reaches the device."""
import os
import re

import numpy as np
import pytest
import torch

import geometry_ref as gr
from patchfusion_b200 import geometry, lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'geometry_case0.npz')
SIZES = ((7, 9), (30, 41), (64, 64))


@pytest.fixture(scope='module')
def golden():
    return np.load(GOLDEN)


@pytest.mark.parametrize('H,W', SIZES)
def test_restatement_matches_reference(golden, H, W):
    tag = '%dx%d' % (H, W)
    depth = golden['depth_' + tag]
    assert np.array_equal(gr.get_intrinsics(H, W), golden['K_' + tag])
    assert np.array_equal(geometry.get_intrinsics(H, W), golden['K_' + tag])
    scale = np.abs(golden['points_' + tag]).max()
    np.testing.assert_allclose(gr.depth_to_points(depth), golden['points_' + tag], rtol=1e-12, atol=1e-12 * scale)
    np.testing.assert_allclose(gr.depth_to_points(depth, golden['R_' + tag], golden['t_' + tag]),
                               golden['points_rt_' + tag], rtol=1e-12, atol=1e-12 * scale)
    tri, tri_m = gr.create_triangles(H, W), gr.create_triangles(H, W, golden['mask_' + tag])
    assert tri.dtype == golden['tri_' + tag].dtype and np.array_equal(tri, golden['tri_' + tag])
    assert np.array_equal(tri_m, golden['tri_mask_' + tag]) and len(tri_m) > 0


def test_golden_is_small():
    assert os.path.getsize(GOLDEN) < 1 << 20


def test_edge_mask_restatement_is_np_gradient():
    """the host mask on a hand-computed case: one-sided differences at the borders, central / 2 inside"""
    d = np.array([[1, 2, 4], [1, 2, 4], [1, 2, 9]], dtype=np.float32)
    gx = np.array([[1, 1.5, 2], [1, 1.5, 2], [1, 4, 7]], dtype=np.float32)
    gy = np.array([[0, 0, 0], [0, 0, 2.5], [0, 0, 5]], dtype=np.float32)
    assert np.array_equal(gr.gradient_norm(d), np.hypot(gy, gx))
    assert np.array_equal(gr.edge_mask(d, 2.0), np.hypot(gy, gx) <= 2)
    d[0, 0], d[0, 1], d[1, 1] = np.nan, 0.0, -1.0
    m = gr.edge_mask(d, 100.0)
    assert not m[0, 0] and not m[0, 1] and not m[1, 1] and not m[1, 0]     # (1, 0)'s y-gradient reads the NaN
    assert m[2, 2]


def test_mesh_scan_block_matches_header():
    src = open(os.path.join(ROOT, 'include', 'pf_b200.h')).read()
    assert int(re.search(r'#define\s+PF_MESH_SCAN_BLOCK\s+(\d+)', src).group(1)) == lib.MESH_SCAN_BLOCK


def _mesh(n, nf, seed=0):
    rng = np.random.default_rng(seed)
    v = rng.normal(size=(n, 3)).astype(np.float32)
    c = rng.integers(0, 256, (n, 3), dtype=np.uint8)
    f = rng.integers(0, max(n, 1), (nf, 3)).astype(np.int32)
    return v, c, f


@pytest.mark.parametrize('n,nf', [(17, 23), (0, 0), (5, 0), (1000, 1)])
@pytest.mark.parametrize('with_color', [True, False])
def test_ply_roundtrip(tmp_path, n, nf, with_color):
    v, c, f = _mesh(n, nf)
    path = str(tmp_path / 'm.ply')
    geometry.write_ply(path, v, c if with_color else None, f)
    r = gr.read_ply(path)
    assert r['counts'] == (n, nf)
    assert ('element vertex %d' % n) in r['header'] and ('element face %d' % nf) in r['header']
    assert np.array_equal(r['vertices'], v) and np.array_equal(r['faces'], f)
    assert (r['colors'] is None) == (not with_color)
    if with_color:
        assert np.array_equal(r['colors'], c)
    # CPU tensors and the reference's int64 faces give the same bytes
    path2 = str(tmp_path / 'm2.ply')
    geometry.write_ply(path2, torch.from_numpy(v), torch.from_numpy(c) if with_color else None, f.astype(np.int64))
    assert open(path, 'rb').read() == open(path2, 'rb').read()


def test_ply_without_faces(tmp_path):
    v, c, _ = _mesh(9, 0)
    path = str(tmp_path / 'p.ply')
    geometry.write_ply(path, v, c, None)
    assert gr.read_ply(path)['counts'] == (9, 0)


def test_ply_rejects_out_of_range_faces(tmp_path):
    v, c, f = _mesh(4, 2)
    with pytest.raises(ValueError):
        geometry.write_ply(str(tmp_path / 'x.ply'), v, c, f.astype(np.int64) + 2 ** 31)


@pytest.mark.parametrize('h,w', [(2 ** 16, 2 ** 15), (1, 10), (10, 1), (0, 5), (46341, 46341)])
def test_create_triangles_rejects_bad_sizes(h, w):
    with pytest.raises(ValueError):
        geometry.create_triangles(h, w)


@pytest.mark.parametrize('shape', [(5, 6), (6, 5), (30,), (1, 5, 7)])
def test_create_triangles_rejects_mask_shape(shape):
    with pytest.raises(ValueError, match='shape'):
        geometry.create_triangles(5, 7, torch.ones(shape, dtype=torch.bool))


@pytest.mark.parametrize('flat', [False, True])
def test_create_triangles_rejects_mask_on_host(flat):
    m = torch.ones((5, 7), dtype=torch.bool)
    with pytest.raises(ValueError, match='CUDA'):
        geometry.create_triangles(5, 7, m.reshape(-1) if flat else m)


@pytest.mark.parametrize('fn', ['points', 'edges', 'mesh'])
def test_host_depth_is_refused(fn):
    d = torch.ones(1, 8, 8)
    with pytest.raises(ValueError, match='CUDA'):
        {'points': lambda: geometry.depth_to_points(d), 'edges': lambda: geometry.depth_edges_mask(d, 1.0),
         'mesh': lambda: geometry.depth_to_mesh(d)}[fn]()


def test_pose_is_validated():
    with pytest.raises(ValueError):
        geometry._rt(np.eye(4), None)
    with pytest.raises(ValueError):
        geometry._rt(None, np.zeros(4))
    rt = geometry._rt(np.arange(9.0).reshape(3, 3), [1, 2, 3])
    assert rt == [float(v) for v in range(9)] + [1.0, 2.0, 3.0]
    assert geometry._rt(None, None) is None
