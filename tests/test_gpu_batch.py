"""Batched inference (several images per forward): every check is bit-exact (max diff == 0.0) against single-image
calls made in order from the same `random` state, unless a tolerance is stated.

Kernel level: the indexed crop-resize / ROI crop-zoom against per-image calls of the single-image entry points, and
pf_g2l_forward at B = 3 against three B = 1 calls.  End to end: PatchFusion (vits fixture weights) in m1 / m2 / r4 with
micro-batches that straddle images, CUDA graphs off / replayed / alternating batch sizes, emulated tile sharding in both
coarse modes, BaselinePretrain's fine target, the Tester at batch_size 3, vitl 4K P49 at B = 2, and a real NCCL
sharded batch when more than one GPU is visible."""
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_DEPTH = 80.0


def _same(tag, a, b):
    assert a.shape == b.shape, (tag, a.shape, b.shape)
    d = (a.float() - b.float()).abs().max().item()
    print('%s: max diff %.3e' % (tag, d))
    assert torch.isfinite(a.float()).all(), tag + ': non-finite values in the first operand'
    assert torch.isfinite(b.float()).all(), tag + ': non-finite values in the second operand'
    assert d == 0.0, tag


@pytest.fixture(scope='module')
def vits(cuda):
    from oracle.make_golden import case_inputs, load_parts
    from patchfusion_b200.model import PatchFusion
    case = json.load(open(os.path.join(GOLD, 'vits_case0.json')))
    cfg, sd, img0 = case_inputs(case)
    shape = tuple(case['image_raw_shape'])
    imgs = [img0] + [torch.rand(1, 3, *shape, generator=torch.Generator().manual_seed(s)) for s in (101, 202)]
    model = PatchFusion(cfg)
    model.load_state_dict(sd, strict=True)
    model = model.to(cuda).eval()
    imgs = torch.cat(imgs).to(cuda)
    return dict(case=case, cfg=cfg, sd=sd, model=model, imgs=imgs, lr=model.make_lr(imgs),
                gold=load_parts(os.path.join(GOLD, 'vits_case0')))


def _sequential(model, lr, imgs, seed, **kw):
    """B single-image calls in order from one `random` state"""
    random.seed(seed)
    return torch.cat([model(mode='infer', image_lr=lr[b:b + 1], image_hr=imgs[b:b + 1], **kw)[0].clone()
                      for b in range(imgs.shape[0])])


def _batched(model, lr, imgs, seed, **kw):
    random.seed(seed)
    y, info = model(mode='infer', image_lr=lr, image_hr=imgs, **kw)
    assert info['depth_pred'] is y and info['rgb'] is lr
    return y.clone()


# ---------------------------------------------------------------------------------------------------- kernel level
def test_crop_resize_batched(cuda):
    from patchfusion_b200 import ops
    g = torch.Generator().manual_seed(0)
    B, H, W, th, tw, ph, pw = 3, 120, 200, 60, 100, 56, 70
    img = torch.rand(B, 3, H, W, generator=g).to(cuda)
    org = [(0, 0), (60, 100), (30, 50), (0, 100), (59, 99), (17, 3), (60, 0)]
    which = [2, 0, 1, 1, 2, 0, 2]
    T = len(org)
    o = torch.tensor(org, dtype=torch.int32, device=cuda)
    idx = torch.tensor(which, dtype=torch.int32, device=cuda)
    got = torch.full((T, 3, ph, pw), float('nan'), device=cuda)
    ops.call('pf_crop_resize_batched', img, H, W, o, idx, T, th, tw, ph, pw, got, ops.stream_ptr())
    for t in range(T):
        one = torch.empty((1, 3, ph, pw), device=cuda)
        ops.call('pf_crop_resize', img[which[t]].contiguous(), H, W, o[t:t + 1].contiguous(), 1, th, tw, ph, pw, one,
                 ops.stream_ptr())
        _same('crop_resize tile %d (image %d)' % (t, which[t]), got[t:t + 1], one)
    old, new = torch.empty_like(got), torch.empty_like(got)
    ops.call('pf_crop_resize', img[0].contiguous(), H, W, o, T, th, tw, ph, pw, old, ops.stream_ptr())
    ops.call('pf_crop_resize_batched', img, H, W, o, None, T, th, tw, ph, pw, new, ops.stream_ptr())
    _same('crop_resize NULL index == pf_crop_resize', new, old)


@pytest.mark.parametrize('f32', [False, True])
def test_roi_crop_zoom_batched(cuda, f32):
    import ctypes as C
    from patchfusion_b200 import ops
    g = torch.Generator().manual_seed(1)
    B, h, w, Cc, ld = 3, 14, 19, 40, 48
    if f32:
        feat = torch.rand(B, h, w, generator=g).to(cuda)
        Cc, ld = 1, 1
    else:
        feat = torch.zeros(B, h, w, ld, dtype=torch.bfloat16, device=cuda)
        feat[..., :Cc] = torch.randn(B, h, w, Cc, generator=g).to(cuda, torch.bfloat16)
    P = (392, 518)
    boxes = torch.tensor([[0, 0, 259, 196], [129.5, 98, 388.5, 294], [259, 196, 518, 392], [10.25, 3.5, 300, 200],
                          [0, 0, 518, 392]], dtype=torch.float32, device=cuda)
    which = [1, 2, 0, 2, 1]
    T = boxes.shape[0]
    idx = torch.tensor(which, dtype=torch.int32, device=cuda)
    oshape = (T, h, w) if f32 else (T, h, w, ld)
    got = torch.zeros(oshape, dtype=feat.dtype, device=cuda)      # pad channels are not written
    ops.call('pf_roi_crop_zoom_batched', feat, int(f32), h, w, ops.pad_to(Cc, 8) if not f32 else 1, ld, idx, boxes, T,
             C.c_float(h / P[0]), got, ld, 0, ops.stream_ptr())
    for t in range(T):
        one = torch.zeros((1,) + oshape[1:], dtype=feat.dtype, device=cuda)
        ops.roi_crop_zoom(feat[which[t]].contiguous() if f32 else feat[which[t]:which[t] + 1].contiguous(), Cc,
                          boxes[t:t + 1].contiguous(), h / P[0], one)
        _same('roi_crop_zoom %s box %d (image %d)' % ('f32' if f32 else 'bf16', t, which[t]), got[t:t + 1], one)
    old = torch.zeros(oshape, dtype=feat.dtype, device=cuda)
    ops.call('pf_roi_crop_zoom', feat, int(f32), h, w, ops.pad_to(Cc, 8) if not f32 else 1, ld, boxes, T,
             C.c_float(h / P[0]), old, ld, 0, ops.stream_ptr())
    new = torch.zeros_like(old)
    ops.call('pf_roi_crop_zoom_batched', feat, int(f32), h, w, ops.pad_to(Cc, 8) if not f32 else 1, ld, None, boxes,
             T, C.c_float(h / P[0]), new, ld, 0, ops.stream_ptr())
    _same('roi_crop_zoom NULL index == pf_roi_crop_zoom', new, old)


def test_g2l_forward_batched(cuda, vits):
    """pf_g2l_forward over B = 3 coarse maps == three B = 1 calls, at every level (each level has its own width, head
    count and so head_dim, and its own padded window grid)"""
    from patchfusion_b200.engine import Map
    eng = vits['model'].engine()
    cd, cf = eng.branch('coarse', vits['lr'].contiguous())
    cf = [Map(m.t.clone(), m.C) for m in cf]
    heads = [(g.C, g.heads) for g in eng.c_fusion.g2l]
    print('G2L levels (C, heads):', heads, 'head_dims', sorted(set(c // h for c, h in heads)))
    batch = [Map(m.t.clone(), m.C) for m in eng.g2l(cf)]
    assert all(m.B == 3 for m in batch)
    for b in range(3):
        one = eng.g2l([Map(m.t[b:b + 1].contiguous(), m.C) for m in cf])
        for i in range(6):
            _same('g2l level %d (C %d, heads %d) image %d' % (i, heads[i][0], heads[i][1], b), batch[i].t[b:b + 1],
                  one[i].t)


# ---------------------------------------------------------------------------------------------------- PatchFusion
@pytest.mark.parametrize('mode', ['m1', 'm2', 'r4'])
def test_patchfusion_batch_equals_sequential(cuda, vits, mode):
    """B = 3 distinct images; process_num 1, 2, 4, 9 so that micro-batches straddle images (m2 has 9 tiles per image)"""
    model, lr, imgs = vits['model'], vits['lr'], vits['imgs']
    for pn in (1, 2, 4, 9):
        want = _sequential(model, lr, imgs, 7, cai_mode=mode, process_num=pn)
        got = _batched(model, lr, imgs, 7, cai_mode=mode, process_num=pn)
        _same('%s process_num %d: B=3 vs 3 x B=1' % (mode, pn), got, want)


@pytest.mark.parametrize('mode', ['m1', 'm2', 'r4'])
def test_patchfusion_batch_image0_vs_reference_fixture(cuda, vits, mode):
    case = vits['case']
    got = _batched(vits['model'], vits['lr'], vits['imgs'], 0, cai_mode=mode, process_num=case['process_num'])
    st = case['sample_stride']
    g = torch.tensor(vits['gold']['infer_' + mode])
    y = got[:1].cpu()[..., ::st, ::st]
    assert y.shape == g.shape
    err = (y - g).abs().max().item()
    print('%s image 0 of B=3 vs reference fixture: max-abs %.3e /max_depth %.3e' % (mode, err, err / MAX_DEPTH))
    assert err / MAX_DEPTH < 1e-3
    assert err / (g.max() - g.min()).item() < 2e-2


def test_graphs_off_replay_and_alternating_batch_sizes(cuda, vits):
    model, lr, imgs = vits['model'], vits['lr'], vits['imgs']
    kw = dict(cai_mode='r4', process_num=2)
    ref = _sequential(model, lr, imgs, 3, **kw)
    model.use_cuda_graphs = False
    try:
        _same('graphs off: B=3', _batched(model, lr, imgs, 3, **kw), ref)
    finally:
        model.use_cuda_graphs = True
    _same('graphs on: B=3 capture', _batched(model, lr, imgs, 3, **kw), ref)
    _same('graphs on: B=3 replay', _batched(model, lr, imgs, 3, **kw), ref)
    random.seed(3)
    for rep in range(2):        # B=1 and B=3 interleaved on one model, from one random stream
        y1 = model(mode='infer', image_lr=lr[:1], image_hr=imgs[:1], **kw)[0].clone()
        y3 = model(mode='infer', image_lr=lr[1:], image_hr=imgs[1:], **kw)[0].clone()
        if rep == 0:
            _same('alternating: B=1 then B=2', torch.cat([y1, y3]), ref)
    _same('after alternation: B=3 replay', _batched(model, lr, imgs, 3, **kw), ref)


@pytest.mark.parametrize('how', ['owner', 'replicate'])
def test_emulated_sharding(cuda, vits, how):
    model, lr, imgs = vits['model'], vits['lr'], vits['imgs']
    model.shard_coarse = how
    try:
        for mode in ('m2', 'r4'):
            want = _sequential(model, lr, imgs, 11, cai_mode=mode, process_num=2)
            for W in (2, 3, 8):
                got = _batched(model, lr, imgs, 11, cai_mode=mode, process_num=2, shard=('emulate', W))
                _same('%s %s emulated world %d: B=3 vs 3 x B=1' % (how, mode, W), got, want)
        model.random_chunk = 3                      # r8 at process_num 2: 8 random tiles per image, chunks of 3
        try:
            want = _sequential(model, lr, imgs, 12, cai_mode='r8', process_num=2)
            for W in (1, 3):
                sh = None if W == 1 else ('emulate', W)
                got = _batched(model, lr, imgs, 12, cai_mode='r8', process_num=2, shard=sh)
                _same('%s r8 chunks of 3, world %d' % (how, W), got, want)
        finally:
            model.random_chunk = 4096
    finally:
        model.shard_coarse = 'owner'


# ---------------------------------------------------------------------------------------------------- BaselinePretrain / Tester
def test_baseline_fine_target_batch(cuda, vits):
    from patchfusion_b200.baseline import BaselinePretrain
    from test_baseline_host import pretrain_model_cfg
    cfg = pretrain_model_cfg(vits['case']['encoder'], 'fine', image_raw_shape=tuple(vits['case']['image_raw_shape']),
                             patch_split_num=tuple(vits['case']['patch_split_num']))
    cfg.pop('type')
    m = BaselinePretrain(**cfg)
    m.load_dict({k[len('fine_branch.'):]: v for k, v in vits['sd'].items() if k.startswith('fine_branch.')})
    m = m.to(cuda).eval()
    imgs = vits['imgs']
    for mode, pn in (('m1', 2), ('m2', 4), ('r4', 3)):
        random.seed(5)
        want = torch.cat([m(mode='infer', image_lr=None, image_hr=imgs[b:b + 1], cai_mode=mode, process_num=pn)[0].clone()
                          for b in range(3)])
        random.seed(5)
        got, info = m(mode='infer', image_lr=None, image_hr=imgs, cai_mode=mode, process_num=pn)
        assert info == {}
        _same('BaselinePretrain fine %s process_num %d: B=3 vs 3 x B=1' % (mode, pn), got, want)


def test_tester_batch_size(cuda, vits, tmp_path):
    from patchfusion_b200.tester import Tester
    model = vits['model']
    H, W = vits['case']['image_raw_shape']
    g = torch.Generator().manual_seed(8)
    rng = np.random.default_rng(3)
    samples = [dict(img_file_basename='s%d' % i, image_u8=rng.integers(0, 256, (H // 2, W // 2, 3), dtype=np.uint8),
                    depth_gt=torch.rand(1, 1, H, W, generator=g) * 2 + 0.2) for i in range(4)]
    split = dict(image_raw_shape=(H, W), patch_split_num=tuple(vits['case']['patch_split_num']))
    res = {}
    for bs in (1, 3):
        d = tmp_path / ('bs%d' % bs)
        res[bs] = Tester(model, work_dir=str(d), save=True, gray_scale=True).run(samples, cai_mode='m2', process_num=4,
                                                                 batch_size=bs, **split)
    assert len(res[1]) == len(res[3]) == 4
    for a, b in zip(res[1], res[3]):
        assert a == b, (a, b)
    for i in range(4):
        for suffix in ('', '_uint16'):
            f1 = (tmp_path / 'bs1' / ('s%d%s.png' % (i, suffix))).read_bytes()
            f3 = (tmp_path / 'bs3' / ('s%d%s.png' % (i, suffix))).read_bytes()
            assert f1 == f3, 's%d%s.png differs between batch_size 1 and 3' % (i, suffix)


# ---------------------------------------------------------------------------------------------------- vitl 4K P49
def test_vitl_4k_p49_batch_of_two(cuda):
    from patchfusion_b200.configs import depth_anything_patchfusion
    from patchfusion_b200.model import PatchFusion
    from patchfusion_b200.params import synthetic_state_dict
    cfg = depth_anything_patchfusion('vitl')
    model = PatchFusion(cfg)
    model.load_state_dict(synthetic_state_dict(cfg, seed=0), strict=True)
    model = model.to(cuda).eval()
    imgs = torch.cat([torch.rand(1, 3, 2160, 3840, generator=torch.Generator().manual_seed(s)) for s in (3, 4)]).to(cuda)
    lr = model.make_lr(imgs)
    want = _sequential(model, lr, imgs, 0, cai_mode='m2', process_num=9)
    got = _batched(model, lr, imgs, 0, cai_mode='m2', process_num=9)
    assert got.shape == (2, 1, 1568, 2072)
    _same('vitl 4K P49 m2 process_num 9: B=2 vs 2 x B=1', got, want)


# ---------------------------------------------------------------------------------------------------- NCCL
def test_nccl_sharded_batch_matches_single_gpu(cuda):
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip('needs >= 2 GPUs')
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', str(n), '--master-addr',
           '127.0.0.1', '--master-port', '29643', os.path.join(ROOT, 'tools', 'check_shard_batch.py')]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=800)
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0
