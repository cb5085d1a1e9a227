"""BaselinePretrain on the CUDA path (vits and vitl) against BaselineOracle executed by torch on the GPU in fp32 (TF32
off) and against the reference fixture vits_baseline0 (oracle/make_golden_baseline.py), plus the bit-exact
invariances of the tile path: micro-batch size, emulated tile sharding, graphs on/off and replay, chunked random
phase, and agreement with PatchFusion's own branch on shared weights.

Tolerance as everywhere here: |d - d_ref| / max_depth(80) < 1e-3 AND |d - d_ref| / (max d_ref - min d_ref) < 2e-2."""
import json
import os
import random

import pytest
import torch
import torch.nn.functional as F

from test_baseline_host import pretrain_model_cfg

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
MAX_DEPTH = 80.0


def _report(tag, got, want):
    got, want = got.float().cpu(), want.float().cpu()
    assert got.shape == want.shape, (tag, got.shape, want.shape)
    err = (got - want).abs().max().item()
    rng = (want.max() - want.min()).item()
    print('%s: max-abs %.3e  /max_depth %.3e  /range %.3e  (range %.3f..%.3f)' %
          (tag, err, err / MAX_DEPTH, err / rng, want.min().item(), want.max().item()))
    assert torch.isfinite(got).all(), tag
    assert err / MAX_DEPTH < 1e-3, tag
    assert err / rng < 2e-2, tag


def _same(tag, a, b):
    d = (a.float() - b.float()).abs().max().item()
    print('%s: max diff %.3e' % (tag, d))
    assert d == 0.0, tag


def _build(target, sd, cuda, **kw):
    from patchfusion_b200.baseline import BaselinePretrain
    cfg = pretrain_model_cfg(sd['enc'], target, **kw)
    cfg.pop('type')
    m = BaselinePretrain(**cfg)
    pre = target + '_branch.'
    m.load_dict({k[len(pre):]: v for k, v in sd['sd'].items() if k.startswith(pre)})
    return cfg, m.to(cuda).eval()


@pytest.fixture(scope='module')
def vits(cuda):
    from oracle.make_golden import case_inputs, load_parts
    case = json.load(open(os.path.join(GOLD, 'vits_baseline0.json')))
    cfg, sd, img = case_inputs(case)
    img2 = torch.rand(1, 3, *case['image_raw_shape'], generator=torch.Generator().manual_seed(case['input_seed'] + 1))
    img3 = torch.rand(1, 3, *case['image_raw_shape'], generator=torch.Generator().manual_seed(99))
    return dict(case=case, pf_cfg=cfg, enc=case['encoder'], sd=sd, sdc={k: v.to(cuda) for k, v in sd.items()},
                imgs=torch.cat([img, img2, img3]).to(cuda), gold=load_parts(os.path.join(GOLD, 'vits_baseline0')),
                split=dict(image_raw_shape=tuple(case['image_raw_shape']),
                           patch_split_num=tuple(case['patch_split_num'])))


def test_coarse_target(cuda, vits):
    """Shipped coarse config (default patch_process_shape (384, 512)), B = 3 at 392x518: oracle, fixture, B = 1
    runs, PatchFusion.coarse_forward on the same weights; then a re-pack at 266x350."""
    from oracle.baseline_oracle import BaselineOracle
    from patchfusion_b200.model import PatchFusion
    v = vits
    cfg, model = _build('coarse', v, cuda)
    orc = BaselineOracle(v['sdc'], cfg, 'coarse')
    lr = F.interpolate(v['imgs'], (392, 518), mode='bilinear', align_corners=True)
    y, info = model(mode='infer', image_lr=lr, image_hr=None)
    y = y.clone()
    assert y.shape == (3, 1, 392, 518) and set(info) == {'rgb', 'depth_pred', 'depth_gt'}
    with torch.no_grad():
        want = orc.infer(lr, None)
    _report('coarse B=3 392x518 vs oracle', y, want)
    st = v['case']['sample_stride']
    _report('coarse 392x518 vs reference fixture', y[:2, :, ::st, ::st], torch.tensor(v['gold']['coarse_392x518']))
    y2, _ = model(mode='infer', image_lr=lr, image_hr=None)            # replayed graph
    _same('coarse replay', y2, y)
    for i in range(3):
        yi, _ = model(mode='infer', image_lr=lr[i:i + 1], image_hr=None)
        _same('coarse image %d: B=3 vs B=1' % i, yi, y[i:i + 1])
    pf = PatchFusion(v['pf_cfg'])
    pf.load_state_dict(v['sd'], strict=True)
    pf = pf.to(cuda).eval()
    for i in range(3):
        d, _ = pf.coarse_forward(lr[i:i + 1])
        _same('coarse image %d vs PatchFusion.coarse_forward' % i, d, y[i:i + 1])
    del pf
    lr2 = F.interpolate(v['imgs'][:2], (266, 350), mode='bilinear', align_corners=True)
    y3, _ = model(mode='infer', image_lr=lr2, image_hr=None)
    assert model.engine((266, 350)).P == (266, 350)
    with torch.no_grad():
        _report('coarse B=2 266x350 (re-packed) vs oracle', y3, orc.infer(lr2, None))
    # the reference's own resizer output (378x518) against the fixture
    lr3 = model.resizer(v['imgs'][:2])
    assert tuple(lr3.shape[-2:]) == (378, 518)
    y4, _ = model(mode='infer', image_lr=lr3, image_hr=None)
    _report('coarse 378x518 vs reference fixture', y4[..., ::st, ::st], torch.tensor(v['gold']['coarse_378x518']))


@pytest.fixture(scope='module')
def fine(cuda, vits):
    from oracle.baseline_oracle import BaselineOracle
    cfg, model = _build('fine', vits, cuda, **vits['split'])
    return dict(cfg=cfg, model=model, orc=BaselineOracle(vits['sdc'], cfg, 'fine'), img=vits['imgs'][:1].contiguous())


@pytest.mark.parametrize('mode', ['m1', 'm2', 'r4'])
def test_fine_target_vs_oracle_and_fixture(cuda, vits, fine, mode):
    pn = vits['case']['process_num']
    random.seed(0)
    y, info = fine['model'](mode='infer', image_lr=None, image_hr=fine['img'], cai_mode=mode, process_num=pn)
    y = y.clone()
    assert info == {}
    random.seed(0)
    with torch.no_grad():
        want = fine['orc'].infer(None, fine['img'], cai_mode=mode, process_num=pn)
    _report('fine %s vs oracle' % mode, y, want)
    st = vits['case']['sample_stride']
    _report('fine %s vs reference fixture' % mode, y[..., ::st, ::st], torch.tensor(vits['gold']['fine_' + mode]))


def test_fine_target_invariances(cuda, fine):
    model, img = fine['model'], fine['img']

    def run(mode='r4', pn=2, **kw):
        random.seed(3)
        y, _ = model(mode='infer', image_lr=None, image_hr=img, cai_mode=mode, process_num=pn, **kw)
        return y.clone()

    base = run('m2', 2)
    for pn in (1, 4, 9):
        _same('m2 process_num %d vs 2' % pn, run('m2', pn), base)
    ref = run()
    _same('r4 replayed', run(), ref)
    for W in (2, 3, 8):
        _same('r4 shard emulate %d' % W, run(shard=('emulate', W)), ref)
    model.use_cuda_graphs = False
    try:
        _same('r4 graphs off', run(), ref)
    finally:
        model.use_cuda_graphs = True
    model.random_chunk = 3                                      # 8 random tiles -> chunks 3, 3, 2
    try:
        _same('r4 random phase in chunks of 3', run(), ref)
        _same('r4 chunks of 3, sharded 3 ways', run(shard=('emulate', 3)), ref)
    finally:
        model.random_chunk = 4096


def test_fine_tile_matches_patchfusion_branch(cuda, vits, fine):
    from patchfusion_b200 import ops
    from patchfusion_b200.model import PatchFusion
    model, img = fine['model'], fine['img']
    pf = PatchFusion(vits['pf_cfg'])
    pf.load_state_dict(vits['sd'], strict=True)
    pf = pf.to(cuda).eval()
    H, W = vits['split']['image_raw_shape']
    h, w = H // 2, W // 2
    ph, pw = model.patch_process_shape
    eng = model.engine()
    tiles = [(h // 2, w // 2), (0, 0)]
    img3 = img[0].contiguous()
    blk = model._compute_phase(eng, 'reg', img3, (H, W, h, w, ph, pw), tiles, 2, None).clone()
    crops = torch.empty((2, 3, ph, pw), device=cuda)
    org = torch.tensor(tiles, dtype=torch.int32, device=cuda)
    ops.call('pf_crop_resize', img3, H, W, org, 2, h, w, ph, pw, crops, ops.stream_ptr())
    d, _ = pf.engine().branch('fine', crops)
    _same('fine tiles vs PatchFusion.engine().branch', blk[:2], d)


def test_random_phase_above_4096_tiles(cuda, fine):
    """r520 at process_num 8: 4160 random tiles, more than one pf_stitch_gather call takes."""
    random.seed(1)
    y, _ = fine['model'](mode='infer', image_lr=None, image_hr=fine['img'], cai_mode='r520', process_num=8)
    torch.cuda.synchronize()
    print('r520 x 8 = 4160 random tiles: out %s range %.3f..%.3f' % (tuple(y.shape), y.min().item(), y.max().item()))
    assert y.shape == (1, 1, 1080, 1920) and torch.isfinite(y).all()


def test_vitl_4k_p49(cuda):
    """Depth-Anything-vitl fine target at 4K, m2 (49 tiles, process_num 9), full canvas against the oracle."""
    from oracle.baseline_oracle import BaselineOracle
    from patchfusion_b200.params import synthetic_state_dict
    pf_cfg = pretrain_model_cfg('vitl', 'fine')
    sd = synthetic_state_dict({'coarse_branch': pf_cfg['coarse_branch'], 'fine_branch': pf_cfg['fine_branch']},
                              seed=0, prefix='fine_branch.')
    cfg, model = _build('fine', dict(enc='vitl', sd=sd), cuda)
    img = torch.rand(1, 3, 2160, 3840, generator=torch.Generator().manual_seed(3)).to(cuda)
    y, _ = model(mode='infer', image_lr=None, image_hr=img, cai_mode='m2', process_num=9)
    y = y.clone()
    assert y.shape == (1, 1, 1568, 2072)
    orc = BaselineOracle({k: v.to(cuda) for k, v in sd.items()}, cfg, 'fine')
    with torch.no_grad():
        want = orc.infer(None, img, cai_mode='m2', process_num=4)
    _report('vitl 4K P49 fine-only (m2)', y, want)


def _spy(model):
    seen, orig = [], model.forward

    def spy(*a, **kw):
        y, info = orig(*a, **kw)
        seen.append(y.clone())
        return y, info
    model.forward = spy
    return seen, orig


def test_tester_drives_both_targets(cuda, vits, fine):
    """Tester.run (make_lr -> model(mode='infer', ...)) on a fine-target model and on a coarse-target model built from
    the shipped coarse config, whose make_lr rounds (384, 512) to 378x518."""
    from patchfusion_b200.tester import Tester
    img = fine['img']
    split = {k: list(v) for k, v in vits['split'].items()}
    seen, orig = _spy(fine['model'])
    try:
        assert Tester(fine['model']).run([{'img_file_basename': 'a', 'image_hr': img}], cai_mode='m2',
                                         process_num=2, **split) == []
    finally:
        del fine['model'].forward
    y, _ = orig(mode='infer', image_lr=None, image_hr=img, cai_mode='m2', process_num=2)
    assert len(seen) == 1
    _same('Tester fine target vs direct call', seen[0], y)
    cfg, coarse = _build('coarse', vits, cuda)
    lr = coarse.make_lr(img)
    assert tuple(lr.shape[-2:]) == (378, 518)
    _report('make_lr vs resizer', lr, coarse.resizer(img))
    seen, orig = _spy(coarse)
    Tester(coarse).run([{'img_file_basename': 'b', 'image_hr': img}], **split)
    assert len(seen) == 1 and seen[0].shape == (1, 1, 378, 518)
    y, _ = orig(mode='infer', image_lr=lr, image_hr=img)
    _same('Tester coarse target vs direct call', seen[0], y)
