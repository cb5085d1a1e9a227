"""BaselinePretrain host side (no GPU): construction from the reference's config schema, state-dict layout, the
branch-only save / load round trip with PatchFusion(load_branch=True), errors, the resizer's rounding, the chunk plan
of the random phase, and the BaselineOracle restatement against the reference fixture vits_baseline0."""
import copy
import json
import os
import random

import numpy as np
import pytest
import torch

from patchfusion_b200.configs import _BRANCH, depth_anything_patchfusion
from patchfusion_b200.params import synthetic_state_dict

GOLD = os.path.join(os.path.dirname(__file__), 'golden')
MAX_DEPTH = 80.0


def pretrain_model_cfg(enc, target, **kw):
    """The model dict of configs/patchfusion_depthanything/depthanything_<enc>_<target>_pretrain_u4k.py (with
    pretrained_resource=None): the fine configs set patch_process_shape=(392, 518), the coarse ones leave the default."""
    br = dict(copy.deepcopy(_BRANCH), midas_model_type=enc, pretrained_resource=None)
    cfg = dict(type='BaselinePretrain', min_depth=1e-3, max_depth=80, target=target, coarse_branch=br,
               fine_branch=copy.deepcopy(br), sigloss=dict(type='SILogLoss'))
    if target == 'fine':
        cfg['patch_process_shape'] = (392, 518)
    cfg.update(kw)
    return cfg


def layout(enc):
    return json.load(open(os.path.join(GOLD, 'state_dict_layout_%s.json' % enc)))


@pytest.mark.parametrize('enc', ['vits', 'vitb', 'vitl'])
@pytest.mark.parametrize('target', ['coarse', 'fine'])
def test_build_model_on_reference_schema(enc, target):
    from estimator.models import build_model
    from estimator.models.baseline_pretrain import BaselinePretrain
    m = build_model(pretrain_model_cfg(enc, target))
    assert isinstance(m, BaselinePretrain) and m.target == target and m.branch == target
    other = 'fine' if target == 'coarse' else 'coarse'
    assert hasattr(m, target + '_branch') and not hasattr(m, other + '_branch')
    assert all(k.startswith(target + '_branch.') for k in m.state_dict())


def test_attribute_style_config():
    from oracle.shims.mmengine.config import ConfigDict
    from estimator.models import build_model
    m = build_model(ConfigDict(pretrain_model_cfg('vits', 'fine')))
    assert m.fine_branch_cfg.type == 'DA-ZoeDepth' and m.patch_process_shape == (392, 518)


@pytest.mark.parametrize('enc', ['vits', 'vitl'])
@pytest.mark.parametrize('target', ['coarse', 'fine'])
def test_layout_is_the_reference_prefix_subset(enc, target):
    from patchfusion_b200.baseline import BaselinePretrain
    cfg = pretrain_model_cfg(enc, target)
    cfg.pop('type')
    sd = BaselinePretrain(**cfg).state_dict()
    want = [(k, v[0], v[1]) for k, v in layout(enc).items() if k.startswith(target + '_branch.')]
    got = [(k, list(v.shape), str(v.dtype).replace('torch.', '')) for k, v in sd.items()]
    assert got == want


def _model(target, enc='vits', seed=0, **kw):
    from patchfusion_b200.baseline import BaselinePretrain
    cfg = pretrain_model_cfg(enc, target, **kw)
    cfg.pop('type')
    return BaselinePretrain(**cfg).init_synthetic_weights(seed)


def test_synthetic_weights_are_the_patchfusion_subset():
    full = synthetic_state_dict(depth_anything_patchfusion('vits'), seed=4)
    for target in ('coarse', 'fine'):
        sd = _model(target, seed=4).state_dict()
        pre = target + '_branch.'
        assert list(sd) == [k for k in full if k.startswith(pre)]
        assert all(torch.equal(sd[k], full[k]) for k in sd)


def test_load_dict_and_get_save_dict():
    m = _model('coarse', seed=1)
    save = m.get_save_dict()
    assert save and not any(k.startswith(('coarse_branch', 'fine_branch')) for k in save)
    assert list(save) == [k[len('coarse_branch.'):] for k in m.state_dict()]
    m2 = _model('coarse', seed=2)
    res = m2.load_dict(save)
    assert not res.missing_keys and not res.unexpected_keys
    assert all(torch.equal(m2.state_dict()['coarse_branch.' + k], v) for k, v in save.items())
    bad = dict(save)
    bad.pop(next(iter(bad)))
    with pytest.raises(RuntimeError):                   # strict=True (BP:123)
        m2.load_dict(bad)
    with pytest.raises(RuntimeError):
        m2.load_dict(dict(save, extra=torch.zeros(1)))


def test_save_files_load_into_patchfusion(tmp_path):
    from patchfusion_b200.model import PatchFusion
    c, f = _model('coarse', seed=5), _model('fine', seed=6)
    paths = []
    for m, name in ((c, 'coarse.pth'), (f, 'fine.pth')):
        paths.append(str(tmp_path / name))
        torch.save({'model_state_dict': m.get_save_dict()}, paths[-1])
    cfg = depth_anything_patchfusion('vits')
    cfg.update(load_branch=True, pretrain_model=paths)
    pf = PatchFusion(cfg)
    sd = pf.state_dict()
    for m, pre in ((c, 'coarse_branch.'), (f, 'fine_branch.')):
        for k, v in m.state_dict().items():
            assert torch.equal(sd[k], v), k
    assert any(k.startswith('guided_fusion.') for k in sd)


def test_errors():
    from patchfusion_b200.baseline import BaselinePretrain
    cfg = pretrain_model_cfg('vits', 'neither')
    cfg.pop('type')
    m = BaselinePretrain(**cfg)
    assert not hasattr(m, 'coarse_branch') and not hasattr(m, 'fine_branch') and not list(m.state_dict())
    with pytest.raises(NotImplementedError):
        m.load_dict({})
    with pytest.raises(NotImplementedError):
        m.get_save_dict()
    with pytest.raises(NotImplementedError):
        m(mode='infer', image_lr=torch.zeros(1, 3, 28, 28), image_hr=torch.zeros(1, 3, 56, 56))
    for target in ('coarse', 'fine'):
        cfg = pretrain_model_cfg('vits', target)
        cfg.pop('type')
        cfg[target + '_branch']['type'] = 'ZoeDepth'
        with pytest.raises(NotImplementedError):
            BaselinePretrain(**cfg)
    m = _model('coarse')
    with pytest.raises(NotImplementedError):
        m(mode='train', image_lr=torch.zeros(1, 3, 28, 28), image_hr=None)
    with pytest.raises(RuntimeError, match='CUDA'):     # CPU model: no fallback
        m(mode='infer', image_lr=torch.zeros(1, 3, 28, 28), image_hr=None)
    with pytest.raises(RuntimeError, match='CUDA'):
        _model('fine')(mode='infer', image_lr=None, image_hr=torch.zeros(1, 3, 2160, 3840))
    with pytest.raises(AssertionError):                 # dinov2 patch_embed: multiple of 14
        m(mode='infer', image_lr=torch.zeros(1, 3, 384, 512), image_hr=None)


def _resize_da_size(size, in_hw, multiple=14):
    """depth_anything/transform.py get_size with keep_aspect_ratio=False, resize_method='minimal'."""
    out = []
    for want, have in zip(size, in_hw):
        out.append(int((np.round(want / have * have / multiple) * multiple).astype(int)))
    return tuple(out)


@pytest.mark.parametrize('pps', [(384, 512), (392, 518), (400, 600), (518, 392)])
def test_resizer_rounds_to_multiples_of_14(pps):
    m = _model('coarse', patch_process_shape=pps)
    img = torch.rand(1, 3, 270, 480)
    out = m.resizer(img)
    assert tuple(out.shape[-2:]) == _resize_da_size(pps, (270, 480))
    assert out.shape[-2] % 14 == 0 and out.shape[-1] % 14 == 0
    if pps == (384, 512):
        assert tuple(out.shape[-2:]) == (378, 518)
    if pps == (392, 518):
        assert tuple(out.shape[-2:]) == (392, 518)
    assert torch.equal(out, torch.nn.functional.interpolate(img, out.shape[-2:], mode='bilinear', align_corners=True))


def test_patchfusion_resizer_unchanged():
    from patchfusion_b200.model import PatchFusion
    pf = PatchFusion(depth_anything_patchfusion('vits'))
    assert tuple(pf.resizer(torch.rand(1, 3, 270, 480)).shape[-2:]) == (392, 518)


def test_random_phase_chunk_plan():
    from patchfusion_b200.model import TiledModel
    assert TiledModel.random_chunk == 4096
    assert TiledModel._chunks(0, 4096) == []
    assert TiledModel._chunks(4096, 4096) == [(0, 4096)]
    assert TiledModel._chunks(8192, 4096) == [(0, 4096), (4096, 8192)]
    assert TiledModel._chunks(9000, 4096) == [(0, 4096), (4096, 8192), (8192, 9000)]
    assert TiledModel._chunks(7, 3) == [(0, 3), (3, 6), (6, 7)]
    for n, s in ((1, 1), (17, 5), (100, 100), (101, 100)):
        ch = TiledModel._chunks(n, s)
        assert ch[0][0] == 0 and ch[-1][1] == n and all(a[1] == b[0] for a, b in zip(ch, ch[1:]))
        assert all(0 < b - a <= s for a, b in ch)


@pytest.fixture(scope='module')
def gold_case():
    from oracle.make_golden import load_parts
    case = json.load(open(os.path.join(GOLD, 'vits_baseline0.json')))
    return case, load_parts(os.path.join(GOLD, 'vits_baseline0'))


def _check(tag, got, want):
    err = (got - want).abs().max().item()
    rng = (want.max() - want.min()).item()
    print('%s: max-abs vs reference fixture %.3e (range %.3f)' % (tag, err, rng))
    assert err / MAX_DEPTH < 1e-3 and err / rng < 2e-2


def test_oracle_against_reference_fixture_coarse(gold_case):
    from oracle.baseline_oracle import BaselineOracle
    from oracle.make_golden import case_inputs
    case, gold = gold_case
    cfg, sd, img = case_inputs(case)
    img2 = torch.rand(1, 3, *case['image_raw_shape'], generator=torch.Generator().manual_seed(case['input_seed'] + 1))
    imgs = torch.cat([img, img2])
    orc = BaselineOracle(sd, pretrain_model_cfg(case['encoder'], 'coarse'), 'coarse')
    torch.set_num_threads(os.cpu_count())
    lr = orc.resizer(imgs)
    assert list(lr.shape[-2:]) == case['lr_sizes'][0] == [378, 518]
    with torch.no_grad():
        y = orc.infer(lr, None)
    st = case['sample_stride']
    _check('coarse 378x518', y[..., ::st, ::st], torch.tensor(gold['coarse_378x518']))


def test_oracle_against_reference_fixture_fine_m1(gold_case):
    from oracle.baseline_oracle import BaselineOracle
    from oracle.make_golden import case_inputs
    case, gold = gold_case
    cfg, sd, img = case_inputs(case)
    mcfg = pretrain_model_cfg(case['encoder'], 'fine', image_raw_shape=case['image_raw_shape'],
                              patch_split_num=case['patch_split_num'])
    orc = BaselineOracle(sd, mcfg, 'fine')
    torch.set_num_threads(os.cpu_count())
    random.seed(0)
    with torch.no_grad():
        y = orc.infer(None, img, cai_mode='m1', process_num=case['process_num'])
    st = case['sample_stride']
    _check('fine m1', y[..., ::st, ::st], torch.tensor(gold['fine_m1']))
