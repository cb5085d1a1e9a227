"""Mixed-geometry batches: images of different sizes, tile grids and modes in one forward.  Every end-to-end check is
bit-exact (max diff == 0.0) against single-image calls made in order from the same `random` state.

Kernel level: pf_crop_resize_multi against pf_crop_resize_batched on equal geometry (bits), against F.interpolate of
each crop on mixed geometry (fp32 tolerance), and rows past T left untouched.  End to end (vits, synthetic weights):
PatchFusion on 1080x1920 2x2, 720x1280 2x4 and 540x960 1x1 over m1 / m2 / r4, the list form of one geometry against
the tensor batch, CUDA graphs off / on with alternating compositions, emulated sharding in both coarse modes,
BaselinePretrain's fine target, the Tester on a mixed stream, and vitl 4K P49 m2 with 1080p m1."""
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]

SHAPES = [((1080, 1920), (2, 2)), ((720, 1280), (2, 4)), ((540, 960), (1, 1))]


def _same(tag, a, b):
    assert a.shape == b.shape, (tag, a.shape, b.shape)
    d = (a.float() - b.float()).abs().max().item()
    print('%s: max diff %.3e' % (tag, d))
    assert torch.isfinite(a.float()).all() and torch.isfinite(b.float()).all(), tag + ': non-finite values'
    assert d == 0.0, tag


def _same_list(tag, got, want):
    assert isinstance(got, list) and len(got) == len(want), tag
    for b, (g, w) in enumerate(zip(got, want)):
        _same('%s image %d' % (tag, b), g, w)


def _cfgs(shapes):
    return [{'image_raw_shape': list(s), 'patch_split_num': list(p)} for s, p in shapes]


@pytest.fixture(scope='module')
def vits(cuda):
    from patchfusion_b200.configs import depth_anything_patchfusion
    from patchfusion_b200.model import PatchFusion
    cfg = depth_anything_patchfusion('vits')
    model = PatchFusion(cfg).init_synthetic_weights(0).to(cuda).eval()
    imgs = [torch.rand(1, 3, *s, generator=torch.Generator().manual_seed(10 + i)).to(cuda)
            for i, (s, _) in enumerate(SHAPES)]
    return dict(cfg=cfg, model=model, imgs=imgs, cfgs=_cfgs(SHAPES), lr=model.make_lr(imgs))


def _sequential(model, lr, imgs, cfgs, modes, seed, **kw):
    """B single-image calls in order from one `random` state"""
    random.seed(seed)
    return [model(mode='infer', image_lr=lr[b:b + 1], image_hr=imgs[b], tile_cfg=cfgs[b], cai_mode=modes[b],
                  **kw)[0].clone() for b in range(len(imgs))]


def _mixed(model, lr, imgs, cfgs, modes, seed, **kw):
    random.seed(seed)
    y, info = model(mode='infer', image_lr=lr, image_hr=imgs, tile_cfg=cfgs, cai_mode=modes, **kw)
    assert info['depth_pred'] is y
    return [t.clone() for t in y]


# ---------------------------------------------------------------------------------------------------- kernel level
def _table(imgs, sizes, dev):
    from patchfusion_b200 import ops
    return ops.crop_table(imgs, sizes, torch.empty((ops.crop_table_bytes(len(imgs)),), dtype=torch.uint8, device=dev))


def test_crop_resize_multi_equals_batched(cuda):
    from patchfusion_b200 import ops
    g = torch.Generator().manual_seed(0)
    B, H, W, th, tw, ph, pw = 3, 120, 200, 60, 100, 56, 70
    img = torch.rand(B, 3, H, W, generator=g).to(cuda)
    org = torch.tensor([(0, 0), (60, 100), (30, 50), (0, 100), (59, 99), (17, 3), (60, 0)], dtype=torch.int32,
                       device=cuda)
    idx = torch.tensor([2, 0, 1, 1, 2, 0, 2], dtype=torch.int32, device=cuda)
    T = org.shape[0]
    want = torch.full((T, 3, ph, pw), float('nan'), device=cuda)
    ops.call('pf_crop_resize_batched', img, H, W, org, idx, T, th, tw, ph, pw, want, ops.stream_ptr())
    got = torch.full((T + 2, 3, ph, pw), -7.0, device=cuda)
    table = _table([img[b:b + 1].contiguous() for b in range(B)], [(th, tw)] * B, cuda)
    ops.crop_resize_multi(table, org, idx, ph, pw, got[:T])
    _same('crop_resize_multi == crop_resize_batched (equal geometry)', got[:T], want)
    assert (got[T:] == -7.0).all(), 'rows past T were written'


def test_crop_resize_multi_mixed_geometry(cuda):
    from patchfusion_b200 import ops
    g = torch.Generator().manual_seed(1)
    ph, pw = 42, 56
    geo = [((120, 200), (60, 100)), ((90, 64), (45, 16)), ((33, 47), (33, 47))]     # (H, W), (th, tw)
    imgs = [torch.rand(1, 3, *hw, generator=g).to(cuda) for hw, _ in geo]
    tiles = [(0, 0, 0), (1, 45, 48), (2, 0, 0), (0, 60, 100), (1, 0, 16), (0, 31, 7), (1, 22, 3)]
    org = torch.tensor([t[1:] for t in tiles], dtype=torch.int32, device=cuda)
    idx = torch.tensor([t[0] for t in tiles], dtype=torch.int32, device=cuda)
    T = len(tiles)
    got = torch.full((T + 3, 3, ph, pw), -7.0, device=cuda)
    ops.crop_resize_multi(_table(imgs, [s for _, s in geo], cuda), org, idx, ph, pw, got[:T])
    assert (got[T:] == -7.0).all(), 'rows past T were written'
    for t, (b, y, x) in enumerate(tiles):
        th, tw = geo[b][1]
        ref = F.interpolate(imgs[b][:, :, y:y + th, x:x + tw], (ph, pw), mode='bilinear', align_corners=True)
        err = (got[t:t + 1] - ref).abs().max().item()
        print('tile %d (image %d, %dx%d crop): max diff vs F.interpolate %.3e' % (t, b, th, tw, err))
        assert err < 1e-5


def test_make_lr_list(cuda, vits):
    model, imgs = vits['model'], vits['imgs']
    _same('make_lr(list) vs per-image make_lr', vits['lr'], torch.cat([model.make_lr(x) for x in imgs]))


# ---------------------------------------------------------------------------------------------------- PatchFusion
@pytest.mark.parametrize('modes', [['m1', 'm2', 'm1'], ['m2', 'r4', 'm1'], ['r4', 'm1', 'm2']])
def test_mixed_batch_equals_sequential(cuda, vits, modes):
    model, lr, imgs, cfgs = vits['model'], vits['lr'], vits['imgs'], vits['cfgs']
    for pn in (2, 9):
        want = _sequential(model, lr, imgs, cfgs, modes, 7, process_num=pn)
        got = _mixed(model, lr, imgs, cfgs, modes, 7, process_num=pn)
        for b, y in enumerate(got):
            RH, RW = 392 * SHAPES[b][1][0], 518 * SHAPES[b][1][1]
            assert y.shape == ((1, 1) + SHAPES[b][0] if modes[b][0] == 'r' else (1, 1, RH, RW))
        _same_list('%s process_num %d: mixed vs sequential' % ('/'.join(modes), pn), got, want)


def test_list_of_one_geometry_equals_tensor_batch(cuda, vits):
    model = vits['model']
    g = torch.Generator().manual_seed(5)
    imgs = [torch.rand(1, 3, 720, 1280, generator=g).to(cuda) for _ in range(3)]
    cfg = {'image_raw_shape': [720, 1280], 'patch_split_num': [2, 4]}
    lr = model.make_lr(torch.cat(imgs))
    for mode in ('m2', 'r4'):
        random.seed(4)
        want = model(mode='infer', image_lr=lr, image_hr=torch.cat(imgs), tile_cfg=cfg, cai_mode=mode,
                     process_num=4)[0].clone()
        got = _mixed(model, lr, imgs, [cfg] * 3, [mode] * 3, 4, process_num=4)
        _same_list('%s list of one geometry vs tensor batch' % mode, got, list(want.split(1)))


def test_graphs_and_alternating_compositions(cuda, vits):
    model, lr, imgs, cfgs = vits['model'], vits['lr'], vits['imgs'], vits['cfgs']
    modes_a, modes_b = ['m2', 'r4', 'm1'], ['m1', 'm1', 'm2']
    kw = dict(process_num=3)
    ref_a = _sequential(model, lr, imgs, cfgs, modes_a, 3, **kw)
    ref_b = _sequential(model, lr[1:], imgs[1:], cfgs[1:], modes_b[1:], 3, **kw)
    ref_t = _sequential(model, lr[:1], imgs[:1], cfgs[:1], ['m2'], 3, **kw)
    model.use_cuda_graphs = False
    try:
        _same_list('graphs off', _mixed(model, lr, imgs, cfgs, modes_a, 3, **kw), ref_a)
    finally:
        model.use_cuda_graphs = True
    for rep in range(3):                # capture, then replays, with other compositions and a plain batch between
        _same_list('composition A, pass %d' % rep, _mixed(model, lr, imgs, cfgs, modes_a, 3, **kw), ref_a)
        _same_list('composition B, pass %d' % rep, _mixed(model, lr[1:], imgs[1:], cfgs[1:], modes_b[1:], 3, **kw),
                   ref_b)
        random.seed(3)
        y = model(mode='infer', image_lr=lr[:1], image_hr=imgs[0], tile_cfg=cfgs[0], cai_mode='m2', **kw)[0]
        _same('plain single image, pass %d' % rep, y, ref_t[0])


@pytest.mark.parametrize('how', ['owner', 'replicate'])
def test_emulated_sharding(cuda, vits, how):
    model, lr, imgs, cfgs = vits['model'], vits['lr'], vits['imgs'], vits['cfgs']
    modes = ['r4', 'm2', 'm1']
    model.shard_coarse = how
    try:
        want = _sequential(model, lr, imgs, cfgs, modes, 11, process_num=2)
        got = _mixed(model, lr, imgs, cfgs, modes, 11, process_num=2, shard=('emulate', 3))
        _same_list('%s emulated world 3' % how, got, want)
        unsharded = _mixed(model, lr, imgs, cfgs, modes, 11, process_num=2)
        _same_list('%s emulated world 3 vs unsharded' % how, got, unsharded)
    finally:
        model.shard_coarse = 'owner'


# ---------------------------------------------------------------------------------------------------- BaselinePretrain / Tester
def test_baseline_fine_target_mixed(cuda, vits):
    from patchfusion_b200.baseline import BaselinePretrain
    from test_baseline_host import pretrain_model_cfg
    cfg = pretrain_model_cfg('vits', 'fine')
    cfg.pop('type')
    m = BaselinePretrain(**cfg).init_synthetic_weights(0).to(cuda).eval()
    imgs, cfgs = vits['imgs'], vits['cfgs']
    modes = ['r2', 'm2', 'm1']
    for pn in (2, 4):
        random.seed(5)
        want = [m(mode='infer', image_lr=None, image_hr=imgs[b], tile_cfg=cfgs[b], cai_mode=modes[b],
                  process_num=pn)[0].clone() for b in range(3)]
        random.seed(5)
        got, info = m(mode='infer', image_lr=None, image_hr=imgs, tile_cfg=cfgs, cai_mode=modes, process_num=pn)
        assert info == {}
        _same_list('BaselinePretrain fine mixed process_num %d' % pn, got, want)


def test_tester_mixed_stream(cuda, vits, tmp_path):
    from patchfusion_b200.tester import Tester
    model = vits['model']
    rng = np.random.default_rng(3)
    g = torch.Generator().manual_seed(8)
    plan = [(SHAPES[0], 'm2'), (SHAPES[2], 'm1'), (SHAPES[1], 'r4'), (SHAPES[0], 'm1'), (SHAPES[1], None)]
    samples = []
    for i, ((shape, split), mode) in enumerate(plan):
        s = dict(img_file_basename='s%d' % i, image_u8=rng.integers(0, 256, (shape[0] // 2, shape[1] // 2, 3),
                                                                     dtype=np.uint8),
                 depth_gt=torch.rand(1, 1, *shape, generator=g) * 2 + 0.2,
                 tile_cfg={'image_raw_shape': list(shape), 'patch_split_num': list(split)})
        if mode is not None:                        # the last sample falls back to the run's cai_mode
            s['cai_mode'] = mode
        samples.append(s)
    res = {}
    for bs in (1, 3):
        random.seed(2)
        res[bs] = Tester(model, work_dir=str(tmp_path / ('bs%d' % bs)), save=True, gray_scale=True).run(
            samples, cai_mode='m2', process_num=4, batch_size=bs)
    assert len(res[1]) == len(res[3]) == len(samples)
    for a, b in zip(res[1], res[3]):
        assert a == b, (a, b)
    for i in range(len(samples)):
        for suffix in ('', '_uint16'):
            f1 = (tmp_path / 'bs1' / ('s%d%s.png' % (i, suffix))).read_bytes()
            f3 = (tmp_path / 'bs3' / ('s%d%s.png' % (i, suffix))).read_bytes()
            assert f1 == f3, 's%d%s.png differs between batch_size 1 and 3' % (i, suffix)


# ---------------------------------------------------------------------------------------------------- vitl
def test_vitl_4k_p49_with_1080p(cuda):
    from patchfusion_b200.configs import depth_anything_patchfusion
    from patchfusion_b200.model import PatchFusion
    model = PatchFusion(depth_anything_patchfusion('vitl')).init_synthetic_weights(0).to(cuda).eval()
    imgs = [torch.rand(1, 3, 2160, 3840, generator=torch.Generator().manual_seed(3)).to(cuda),
            torch.rand(1, 3, 1080, 1920, generator=torch.Generator().manual_seed(4)).to(cuda)]
    cfgs = _cfgs([((2160, 3840), (4, 4)), ((1080, 1920), (2, 2))])
    modes = ['m2', 'm1']
    lr = model.make_lr(imgs)
    want = _sequential(model, lr, imgs, cfgs, modes, 0, process_num=9)
    got = _mixed(model, lr, imgs, cfgs, modes, 0, process_num=9)
    assert got[0].shape == (1, 1, 1568, 2072) and got[1].shape == (1, 1, 784, 1036)
    _same_list('vitl 4K P49 m2 + 1080p 2x2 m1, process_num 9', got, want)
