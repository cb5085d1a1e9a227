"""patchfusion_b200/geometry.py on the GPU (csrc/pf_geom.cu) against the numpy restatement of the reference's
geometry.py in tests/geometry_ref.py: points within fp32 rounding, triangles and colours exactly, the np.gradient vertex
mask bit for bit where the arithmetic is exact, PLY files through a numpy reader, guard bytes after every output and
argument errors raised before any launch."""
import numpy as np
import pytest
import torch

import geometry_ref as gr
from patchfusion_b200 import geometry, lib, ops

pytestmark = pytest.mark.gpu

GUARD = 0xFF


def _depth(H, W, seed, lo=0.5, hi=80.0):
    return np.random.default_rng(seed).uniform(lo, hi, (1, H, W)).astype(np.float32)


def _pose(seed):
    rng = np.random.default_rng(seed)
    k = rng.normal(size=3)
    k /= np.linalg.norm(k)
    a = 0.7
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(a) * Kx + (1 - np.cos(a)) * Kx @ Kx, rng.uniform(-5.0, 5.0, 3)


def _f32_pose(R, t):
    """the fp32 pose the kernel receives, in fp64 for the reference"""
    return R.astype(np.float32).astype(np.float64), t.astype(np.float32).astype(np.float64)


@pytest.mark.parametrize('H,W', [(2, 2), (17, 31), (1080, 1920), (2160, 3840)])
@pytest.mark.parametrize('posed', [False, True])
def test_points_match_fp64(cuda, H, W, posed):
    d = _depth(H, W, H + W)
    R, t = _pose(H) if posed else (None, None)
    got = geometry.depth_to_points(torch.from_numpy(d).to(cuda), R, t).cpu().numpy().astype(np.float64)
    want = gr.depth_to_points(d, *_f32_pose(R, t)) if posed else gr.depth_to_points(d)
    assert got.shape == (H, W, 3)
    err = np.abs(got - want)
    tol = 2.0 ** -20 * np.abs(want) + 1e-6 * d.max()
    print('%dx%d posed=%s: max |err| %.3e, worst err/tol %.3f' % (H, W, posed, err.max(), (err / tol).max()))
    assert (err <= tol).all()


def test_points_batched_and_views(cuda):
    d = torch.from_numpy(np.concatenate([_depth(24, 40, 1), _depth(24, 40, 2)])[:, None]).to(cuda)
    R, t = _pose(3)
    b = geometry.depth_to_points(d, R, t)
    assert b.shape == (2, 24, 40, 3)
    for i in range(2):
        assert torch.equal(b[i], geometry.depth_to_points(d[i], R, t))
    # a depth view at an odd offset takes the scalar path and gives the same bits
    buf = torch.empty(24 * 40 + 1, device=cuda)
    buf[1:].copy_(d[0].reshape(-1))
    assert torch.equal(geometry.depth_to_points(buf[1:].view(1, 24, 40), R, t), b[0])


@pytest.mark.parametrize('H,W', [(17, 31), (64, 96)])
def test_colors_equal_numpy_rounding(cuda, H, W):
    rng = np.random.default_rng(H)
    img = rng.uniform(-0.2, 1.2, (1, 3, H, W)).astype(np.float32)
    ties = ((np.arange(H * W) % 256) + 0.5) / 255.0                 # values whose 255 v lands on or next to a .5
    img[0, 1] = ties.reshape(H, W).astype(np.float32)
    img[0, 2, 0, :4] = [0.0, 1.0, -0.0, np.float32(0.5 / 255)]
    v, c, f = geometry.depth_to_mesh(torch.from_numpy(_depth(H, W, 0)).to(cuda), torch.from_numpy(img).to(cuda))
    assert c.dtype == torch.uint8 and c.shape == (H * W, 3) and v.shape == (H * W, 3)
    assert np.array_equal(c.cpu().numpy(), gr.colors(img))


def _masks(h, w):
    rng = np.random.default_rng(h * w)
    last_row, last_col = np.zeros((h, w), bool), np.zeros((h, w), bool)
    last_row[-1], last_col[:, -1] = True, True
    split = np.ones((h, w), bool)
    split[::2, ::2] = False            # quads missing tl keep only their second triangle, missing br only the first
    return {'random50': rng.random((h, w)) < 0.5, 'none': np.zeros((h, w), bool), 'all': np.ones((h, w), bool),
            'last_row': last_row, 'last_col': last_col, 'split': split, 'dense': rng.random((h, w)) < 0.85}


def _faces(mask_np, h, w, cuda, dtype=torch.bool):
    m = None if mask_np is None else torch.from_numpy(mask_np).to(dtype).to(cuda)
    return geometry.create_triangles(h, w, m, device=cuda)


@pytest.mark.parametrize('h,w', [(2, 2), (3, 2), (17, 31), (64, 65), (1080, 1920)])
def test_triangles_equal_reference(cuda, h, w):
    got = _faces(None, h, w, cuda)
    assert got.dtype == torch.int32 and np.array_equal(got.cpu().numpy().astype(np.int64), gr.create_triangles(h, w))
    for name, m in _masks(h, w).items():
        for dtype in (torch.bool, torch.uint8):
            got = _faces(m, h, w, cuda, dtype).cpu().numpy()
            want = gr.create_triangles(h, w, m)
            assert got.shape == want.shape and np.array_equal(got.astype(np.int64), want), (name, dtype)
    # the split mask really has quads that keep exactly one triangle, of either kind
    s = _masks(h, w)['split'].reshape(-1)
    tri = gr.create_triangles(h, w).reshape(-1, 2, 3)
    kept = s[tri].all(2)
    if h > 2 and w > 2:
        assert (kept[:, 0] & ~kept[:, 1]).any() and (~kept[:, 0] & kept[:, 1]).any()


@pytest.mark.parametrize('masked', [False, True])
def test_triangles_4k(cuda, masked):
    h, w = 2160, 3840
    nb = ops.mesh_scan_blocks(h, w)
    assert nb > 2 ** 16                 # the block-sum scan runs over more than 2^16 blocks
    m = (np.random.default_rng(4).random((h, w)) < 0.5) if masked else None
    got = _faces(m, h, w, cuda).cpu().numpy().astype(np.int64)
    assert np.array_equal(got, gr.create_triangles(h, w, m))


def _ramp(H, W):
    """integer-valued depth: every np.gradient difference and its square are exact"""
    y, x = np.mgrid[0:H, 0:W]
    d = (1 + 3 * y + 2 * x + 40 * ((x > W // 3) & (y > H // 2)) + 7 * (x % 5 == 0)).astype(np.float32)
    d[0, 0], d[H // 2, W // 2], d[-1, -1] = 0.0, -4.0, np.inf
    d[1, 3 % W] = np.nan
    return d[None]


@pytest.mark.parametrize('H,W', [(2, 2), (17, 31), (1080, 1920)])
def test_edge_mask_exact_on_integer_ramp(cuda, H, W):
    d = _ramp(H, W)
    dd = torch.from_numpy(d).to(cuda)
    for T in (0.0, 2.0, 3.6, 3.7, 5.0, 10.0, 25.0, 1e9):
        got = geometry.depth_edges_mask(dd, T)
        assert got.dtype == torch.bool and got.shape == (H, W)
        assert np.array_equal(got.cpu().numpy(), gr.edge_mask(d, T)), T


@pytest.mark.parametrize('H,W', [(17, 31), (1080, 1920)])
def test_edge_mask_random_depth(cuda, H, W):
    d = _depth(H, W, 7, 1.0, 3.0)
    g = gr.gradient_norm(d)
    dd = torch.from_numpy(d).to(cuda)
    for T in (0.05, 0.3, 0.6):
        got = geometry.depth_edges_mask(dd, T).cpu().numpy()
        want = gr.edge_mask(d, T)
        near = np.abs(g - np.float32(T)) <= 4 * np.spacing(np.float32(T))
        assert np.array_equal(got[~near], want[~near]), T
        assert 0 < want.sum() < want.size
        # the triangles of the device mask are the reference's triangles of that mask
        faces = geometry.create_triangles(H, W, geometry.depth_edges_mask(dd, T))
        assert np.array_equal(faces.cpu().numpy().astype(np.int64), gr.create_triangles(H, W, got))


def test_edge_mask_batched(cuda):
    d = np.concatenate([_ramp(20, 30), _depth(20, 30, 1)])[:, None]
    got = geometry.depth_edges_mask(torch.from_numpy(d).to(cuda), 4.0)
    assert got.shape == (2, 20, 30)
    for i in range(2):
        assert np.array_equal(got[i].cpu().numpy(), gr.edge_mask(d[i], 4.0))


def _read_mesh(path):
    r = gr.read_ply(path)
    return r['vertices'], r['colors'], r['faces']


def test_end_to_end_model_mesh_ply(cuda, tmp_path):
    """seeded vits forward -> depth_to_mesh -> write_ply -> numpy reader == host restatement of the same depth; a
    second run writes the same bytes"""
    from patchfusion_b200.configs import depth_anything_patchfusion
    from patchfusion_b200.model import PatchFusion
    model = PatchFusion(depth_anything_patchfusion('vits', (1080, 1920), (2, 2))).init_synthetic_weights(0).to(cuda).eval()
    img = torch.rand(1, 3, 1080, 1920, generator=torch.Generator().manual_seed(0)).to(cuda)
    tile_cfg = dict(image_raw_shape=[1080, 1920], patch_split_num=[2, 2])
    depth, _ = model(mode='infer', image_lr=model.make_lr(img), image_hr=img, tile_cfg=tile_cfg, cai_mode='m1',
                     process_num=2)
    H, W = depth.shape[-2:]                     # the canvas, at the tiles' network resolution
    img = torch.rand(1, 3, H, W, generator=torch.Generator().manual_seed(1)).to(cuda)
    d = depth[0].cpu().numpy()
    T = float(np.median(gr.gradient_norm(d)))
    paths = []
    for run in range(2):
        v, c, f = geometry.depth_to_mesh(depth[0], img, edge_threshold=T)
        paths.append(str(tmp_path / ('mesh%d.ply' % run)))
        geometry.write_ply(paths[-1], v, c, f)
    blob = open(paths[0], 'rb').read()
    assert blob == open(paths[1], 'rb').read()
    rv, rc, rf = _read_mesh(paths[0])
    want = gr.depth_to_points(d)
    assert rv.shape == (H * W, 3)
    assert (np.abs(rv - want.reshape(-1, 3)) <= 2.0 ** -20 * np.abs(want.reshape(-1, 3)) + 1e-6 * d.max()).all()
    assert np.array_equal(rc, gr.colors(img.cpu().numpy()))
    g = gr.gradient_norm(d)
    mask = geometry.depth_edges_mask(depth[0], T).cpu().numpy()
    near = np.abs(g - np.float32(T)) <= 4 * np.spacing(np.float32(T))
    assert np.array_equal(mask[~near], gr.edge_mask(d, T)[~near])
    assert np.array_equal(rf.astype(np.int64), gr.create_triangles(H, W, mask))
    assert 0 < len(rf) < 2 * (H - 1) * (W - 1)
    print('vits %dx%d mesh: %d vertices, %d faces (threshold %.4g), %d bytes' % (H, W, len(rv), len(rf), T, len(blob)))


def test_mesh_batched_and_mixed_list(cuda):
    a, b = _depth(16, 24, 1), _depth(16, 24, 2)
    img = torch.rand(2, 3, 16, 24, generator=torch.Generator().manual_seed(1)).to(cuda)
    batch = torch.from_numpy(np.concatenate([a, b])[:, None]).to(cuda)
    meshes = geometry.depth_to_mesh(batch, img, edge_threshold=5.0)
    for i, (v, c, f) in enumerate(meshes):
        v1, c1, f1 = geometry.depth_to_mesh(batch[i], img[i:i + 1].contiguous(), edge_threshold=5.0)
        assert torch.equal(v, v1) and torch.equal(c, c1) and torch.equal(f, f1)
    mixed = geometry.depth_to_mesh([torch.from_numpy(_depth(9, 13, 3)).to(cuda), batch[0]])
    assert [m[0].shape[0] for m in mixed] == [9 * 13, 16 * 24] and mixed[0][1] is None
    assert np.array_equal(mixed[0][2].cpu().numpy().astype(np.int64), gr.create_triangles(9, 13))


@pytest.mark.parametrize('n,nf', [(37, 41), (16, 16), (1, 0), (0, 0), (100003, 200001)])
@pytest.mark.parametrize('with_color', [True, False])
def test_ply_device_bytes_equal_host_bytes(cuda, tmp_path, n, nf, with_color):
    rng = np.random.default_rng(n + nf)
    v = rng.normal(size=(n, 3)).astype(np.float32)
    c = rng.integers(0, 256, (n, 3), dtype=np.uint8) if with_color else None
    f = rng.integers(0, max(n, 1), (nf, 3)).astype(np.int32)
    dev = [None if a is None else torch.from_numpy(a).to(cuda) for a in (v, c, f)]
    geometry.write_ply(str(tmp_path / 'd.ply'), *dev)
    geometry.write_ply(str(tmp_path / 'h.ply'), v, c, f)
    assert open(tmp_path / 'd.ply', 'rb').read() == open(tmp_path / 'h.ply', 'rb').read()
    rv, rc, rf = _read_mesh(str(tmp_path / 'd.ply'))
    assert np.array_equal(rv, v) and np.array_equal(rf, f) and (rc is None) == (c is None)


def _poisoned(n, dtype, cuda, extra=4096):
    """a buffer of n elements of dtype followed by `extra` guard bytes, all 0xFF"""
    es = torch.empty((), dtype=dtype).element_size()
    raw = torch.full((n * es + extra,), GUARD, dtype=torch.uint8, device=cuda)
    return raw, raw[:n * es].view(dtype)


def _guard_ok(raw, n_bytes):
    return bool((raw[n_bytes:] == GUARD).all())


@pytest.mark.parametrize('H,W', [(17, 31), (64, 96)])
def test_guard_bytes_points_colors_mask(cuda, H, W):
    n = H * W
    d = torch.from_numpy(_depth(H, W, 5)).to(cuda)
    img = torch.rand(1, 3, H, W, generator=torch.Generator().manual_seed(2)).to(cuda)
    praw, p = _poisoned(3 * n, torch.float32, cuda)
    craw, c = _poisoned(3 * n, torch.uint8, cuda)
    mraw, m = _poisoned(n, torch.uint8, cuda)
    R, t = _pose(1)
    ops.depth_to_points(d, geometry._inv_f(W), geometry._rt(R, t), img, p.view(n, 3), c.view(n, 3))
    ops.depth_edge_mask(d, 10.0, m.view(H, W))
    torch.cuda.synchronize()
    assert _guard_ok(praw, 12 * n) and _guard_ok(craw, 3 * n) and _guard_ok(mraw, n)
    assert torch.equal(p.view(H, W, 3), geometry.depth_to_points(d, R, t))
    assert torch.equal(m.view(H, W).bool(), geometry.depth_edges_mask(d, 10.0))


@pytest.mark.parametrize('h,w', [(17, 31), (300, 257)])
def test_guard_bytes_triangles(cuda, h, w):
    mask = torch.from_numpy(np.random.default_rng(h).random((h, w)) < 0.6).to(cuda)
    want = gr.create_triangles(h, w, mask.cpu().numpy())
    n, nq = len(want), (h - 1) * (w - 1)
    nb = ops.mesh_scan_blocks(h, w)
    fraw, flags = _poisoned(nq, torch.uint8, cuda)
    oraw, offs = _poisoned(nb + 1, torch.int64, cuda)
    ops.mesh_quad_counts(mask, h, w, flags, offs)
    assert int(offs[nb].item()) == n
    for cap in (n, n - 7):                       # the full count, and a buffer too small: rows past cap stay untouched
        traw, faces = _poisoned(3 * cap, torch.int32, cuda)
        ops.mesh_triangles(flags, offs, h, w, faces.view(cap, 3))
        torch.cuda.synchronize()
        assert _guard_ok(traw, 12 * cap), cap
        assert np.array_equal(faces.view(cap, 3).cpu().numpy().astype(np.int64), want[:cap])
    assert _guard_ok(fraw, nq) and _guard_ok(oraw, 8 * (nb + 1))
    araw, allf = _poisoned(6 * nq, torch.int32, cuda)
    ops.mesh_triangles(None, None, h, w, allf.view(2 * nq, 3))
    torch.cuda.synchronize()
    assert _guard_ok(araw, 24 * nq)
    assert np.array_equal(allf.view(-1, 3).cpu().numpy().astype(np.int64), gr.create_triangles(h, w))


@pytest.mark.parametrize('n', [1, 15, 16, 1001])
def test_guard_bytes_ply_records(cuda, n):
    rng = np.random.default_rng(n)
    v = torch.from_numpy(rng.normal(size=(n, 3)).astype(np.float32)).to(cuda)
    c = torch.from_numpy(rng.integers(0, 256, (n, 3), dtype=np.uint8)).to(cuda)
    f = torch.from_numpy(rng.integers(0, n, (n, 3)).astype(np.int32)).to(cuda)
    vraw, vb = _poisoned(15 * n, torch.uint8, cuda)
    fraw, fb = _poisoned(13 * n, torch.uint8, cuda)
    ops.ply_pack_vertices(v, c, vb)
    ops.ply_pack_faces(f, fb)
    torch.cuda.synchronize()
    assert _guard_ok(vraw, 15 * n) and _guard_ok(fraw, 13 * n)
    hv, hf = geometry._pack_host(v.cpu().numpy(), c.cpu().numpy(), f.cpu().numpy())
    assert np.array_equal(vb.cpu().numpy(), hv) and np.array_equal(fb.cpu().numpy(), hf)


def test_errors_raise_before_any_launch(cuda):
    d = torch.from_numpy(_depth(8, 12, 0)).to(cuda)
    img = torch.rand(1, 3, 8, 12, device=cuda)
    mask = torch.ones(8, 12, dtype=torch.bool, device=cuda)
    v, c, f = geometry.depth_to_mesh(d, img)
    torch.cuda.synchronize()
    bad = [
        (TypeError, lambda: geometry.depth_to_points(d.double())),
        (ValueError, lambda: geometry.depth_to_points(d.cpu())),
        (ValueError, lambda: geometry.depth_to_points(d.transpose(1, 2))),
        (TypeError, lambda: geometry.depth_edges_mask(d.half(), 1.0)),
        (ValueError, lambda: geometry.depth_edges_mask(d[:, :, ::2], 1.0)),
        (ValueError, lambda: geometry.depth_edges_mask(d[:, :1], 1.0)),
        (ValueError, lambda: geometry.create_triangles(8, 12, mask.t())),
        (TypeError, lambda: geometry.create_triangles(8, 12, mask.float())),
        (ValueError, lambda: geometry.create_triangles(8, 12, mask.cpu())),
        (ValueError, lambda: geometry.create_triangles(12, 8, mask)),
        (TypeError, lambda: geometry.depth_to_mesh(d, img.double())),
        (ValueError, lambda: geometry.depth_to_mesh(d, img.cpu())),
        (ValueError, lambda: geometry.depth_to_mesh(d, img[:, :, :4])),
        (ValueError, lambda: geometry.depth_to_mesh(d, img.transpose(2, 3).contiguous().transpose(2, 3))),
        (ValueError, lambda: geometry.write_ply('/nonexistent/x.ply', v.t(), c, f)),
        (TypeError, lambda: geometry.write_ply('/nonexistent/x.ply', v, c.int(), f)),
        (TypeError, lambda: geometry.write_ply('/nonexistent/x.ply', v, c, f.long())),
        (ValueError, lambda: geometry.write_ply('/nonexistent/x.ply', v, c.cpu(), f)),
    ]
    for i, (exc, fn) in enumerate(bad):
        before = lib.launch_count()
        with pytest.raises(exc):
            fn()
        assert lib.launch_count() == before, i
