"""BaselinePretrain's calibrated FP8 keys without a GPU: branch_vit_precision / branch_dpt_precision and their tables for
both targets (vits and vitl), their names against PatchFusion's, the state dict, PatchFusion's keys still ignored next to
them, and the config + checkpoint pair the calibration tool writes, loaded back through load_config and build_model."""
import math
import os

import numpy as np
import pytest
import torch

from test_baseline_host import pretrain_model_cfg

TARGETS = ['coarse', 'fine']
ENCODERS = ['vits', 'vitl']


def _cfg(enc, target, **kw):
    cfg = pretrain_model_cfg(enc, target, **kw)
    cfg.pop('type')
    return cfg


def _build(enc, target, **kw):
    from patchfusion_b200.baseline import BaselinePretrain
    return BaselinePretrain(**_cfg(enc, target, **kw))


def _names(enc, target, kind):
    from patchfusion_b200.params import dpt_fp8_layers, vit_fp8_layers
    f = vit_fp8_layers if kind == 'vit' else dpt_fp8_layers
    return f(_cfg(enc, target), (target,))


def _table(enc, target, kind, v=1.5):
    return {k: v + 0.125 * i for i, k in enumerate(_names(enc, target, kind))}


def _layout(m):
    return [(k, tuple(v.shape), v.dtype) for k, v in m.state_dict().items()]


@pytest.mark.parametrize('enc', ENCODERS)
def test_names_are_patchfusion_slices(enc):
    from patchfusion_b200.configs import depth_anything_patchfusion
    from patchfusion_b200.params import dpt_fp8_layers, vit_fp8_layers
    pf = depth_anything_patchfusion(enc)
    depth = {'vits': 12, 'vitl': 24}[enc]
    for target in TARGETS:
        vit, dpt = _names(enc, target, 'vit'), _names(enc, target, 'dpt')
        assert vit == tuple(k for k in vit_fp8_layers(pf) if k.startswith(target + '.'))
        assert dpt == tuple(k for k in dpt_fp8_layers(pf) if k.startswith(target + '.'))
        assert len(vit) == 3 * depth and len(dpt) == 19
    # PatchFusion's own lists are unchanged: both branches, coarse first
    assert vit_fp8_layers(pf) == _names(enc, 'coarse', 'vit') + _names(enc, 'fine', 'vit')
    assert dpt_fp8_layers(pf) == _names(enc, 'coarse', 'dpt') + _names(enc, 'fine', 'dpt')


@pytest.mark.parametrize('enc', ENCODERS)
@pytest.mark.parametrize('target', TARGETS)
def test_precisions(enc, target):
    for vp in ('bf16', 'fp8_static'):
        for dp in ('bf16', 'fp8_static'):
            m = _build(enc, target, branch_vit_precision=vp, branch_dpt_precision=dp)
            assert (m.branch_vit_precision, m.branch_dpt_precision) == (vp, dp)
            assert m.branch_vit_fp8_amax is None and m.branch_dpt_fp8_amax is None and callable(m.calibrate_fp8)
    for key in ('branch_vit_precision', 'branch_dpt_precision'):
        for bad in ('fp8', 'FP8_STATIC', 'e5m2', 'fp16', None):
            with pytest.raises(ValueError, match=key):
                _build(enc, target, **{key: bad})


@pytest.mark.parametrize('enc', ENCODERS)
@pytest.mark.parametrize('target', TARGETS)
@pytest.mark.parametrize('kind', ['vit', 'dpt'])
def test_table_validation(enc, target, kind):
    key = 'branch_%s_fp8_amax' % kind
    prec = 'branch_%s_precision' % kind
    other = 'fine' if target == 'coarse' else 'coarse'
    good = _table(enc, target, kind)
    for p in ('fp8_static', 'bf16'):
        m = _build(enc, target, **{prec: p, key: good})
        assert getattr(m, key) == good
    zero = dict(good)
    first = next(iter(good))
    zero[first] = 0
    zero[list(good)[1]] = np.float32(2.5)
    _build(enc, target, **{prec: 'fp8_static', key: zero})
    missing = dict(good)
    del missing[list(good)[-1]]
    bads = [missing, dict(good, extra=1.0), dict(good, **_table(enc, other, kind)),
            dict(good, **{other + first[len(target):]: 1.0}), {k.replace(target, other, 1): v for k, v in good.items()},
            dict(good, **{first: float('nan')}), dict(good, **{first: math.inf}), dict(good, **{first: -math.inf}),
            dict(good, **{first: -1e-3}), dict(good, **{first: '3.0'}), dict(good, **{first: None}),
            dict(good, **{first: True}), [1.0] * len(good), 'table', 2.0]
    for bad in bads:
        for p in ('fp8_static', 'bf16'):
            with pytest.raises(ValueError, match=key):
                _build(enc, target, **{prec: p, key: bad})


@pytest.mark.parametrize('target', TARGETS)
def test_state_dict_unchanged(target):
    want = _layout(_build('vits', target))
    m = _build('vits', target, branch_vit_precision='fp8_static', branch_vit_fp8_amax=_table('vits', target, 'vit'),
               branch_dpt_precision='fp8_static', branch_dpt_fp8_amax=_table('vits', target, 'dpt'))
    assert _layout(m) == want
    a = _build('vits', target).init_synthetic_weights(3).get_save_dict()
    b = m.init_synthetic_weights(3).get_save_dict()
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    m.load_dict(a)


@pytest.mark.parametrize('target', TARGETS)
def test_patchfusion_keys_still_ignored(target):
    """PatchFusion's keys, any value, next to the baseline's own: the same model as with the new keys alone"""
    from test_fp8_dpt_host import _table as pf_dpt_table
    own = dict(branch_vit_precision='fp8_static', branch_vit_fp8_amax=_table('vits', target, 'vit'))
    want = _build('vits', target, **own)
    for ignored in (dict(vit_precision='bogus', vit_fp8_amax={'bogus': -1}, dpt_precision='fp8_static',
                         dpt_fp8_amax=pf_dpt_table(), fusion_precision='nope', fusion_fp8_amax=[1]),
                    dict(vit_precision='fp8_static', vit_fp8_amax=None, dpt_precision=None)):
        m = _build('vits', target, **own, **ignored)
        assert _layout(m) == _layout(want)
        assert m._fp8_cfg() == want._fp8_cfg()
        assert m.branch_dpt_precision == 'bf16' and m.branch_dpt_fp8_amax is None


def test_without_table_and_bf16_refusals():
    """no table still builds; calibrate_fp8 refuses a model with neither switch on, before touching a device"""
    for target in TARGETS:
        m = _build('vits', target, branch_dpt_precision='fp8_static')
        assert m._fp8_cfg() == {'dpt_precision': 'fp8_static', 'dpt_fp8_amax': None}
        assert _build('vits', target)._fp8_cfg() == {}
        with pytest.raises(ValueError, match='branch_vit_precision'):
            _build('vits', target).calibrate_fp8(None, None)
        with pytest.raises(RuntimeError, match='CUDA'):
            m.calibrate_fp8(torch.zeros(1, 3, 392, 518), torch.zeros(1, 3, 392, 518))


@pytest.mark.parametrize('target', TARGETS)
def test_written_pair_loads_back(tmp_path, target):
    """save_baseline (the calibration tool's writing step): the config file reads back through load_config with the
    tables in its model dict, and build_model + load_dict of the .pth gives the same weights, as tools/test.py builds it"""
    from patchfusion_b200.baseline import save_baseline
    from patchfusion_b200.config import load_config
    from patchfusion_b200.evaluate import build_model
    vt = {k: float(np.float32(v) / np.float32(7.0)) for k, v in _table('vits', target, 'vit').items()}
    dt = _table('vits', target, 'dpt', 0.75)
    m = _build('vits', target, branch_vit_precision='fp8_static', branch_vit_fp8_amax=vt,
               branch_dpt_precision='fp8_static', branch_dpt_fp8_amax=dt).init_synthetic_weights(5)
    cfg = {'model': pretrain_model_cfg('vits', target), 'seed': 5621, 'work_dir': './work_dir/x',
           'val_dataloader': {'batch_size': 1, 'dataset': {'type': 'UnrealStereo4kDataset', 'mode': 'infer',
                                                           'data_root': 'data', 'split': 'splits/test.txt',
                                                           'min_depth': 1e-3, 'max_depth': 80, 'transform_cfg':
                                                           {'network_process_size': [384, 512]}}}}
    name = 'depthanything_vits_%s_pretrain_u4k' % target
    py, pth = save_baseline(m, cfg, str(tmp_path / 'out'), name)
    assert (py, pth) == (str(tmp_path / 'out' / (name + '.py')), str(tmp_path / 'out' / (name + '.pth')))
    back = load_config(py)
    assert back['model']['branch_vit_fp8_amax'] == vt and back['model']['branch_dpt_fp8_amax'] == dt
    assert back['model']['branch_vit_precision'] == back['model']['branch_dpt_precision'] == 'fp8_static'
    assert back['val_dataloader'] == cfg['val_dataloader'] and back['seed'] == 5621
    assert tuple(back['model']['coarse_branch']['n_attractors']) == tuple(cfg['model']['coarse_branch']['n_attractors'])
    m2 = build_model(back, pth)
    assert type(m2) is type(m) and m2.target == target
    assert m2.branch_vit_fp8_amax == vt and m2.branch_dpt_fp8_amax == dt and m2._fp8_cfg() == m._fp8_cfg()
    a, b = m.state_dict(), m2.state_dict()
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    assert sorted(os.listdir(tmp_path / 'out')) == sorted([name + '.py', name + '.pth'])


def test_save_config_refuses_what_does_not_load_back(tmp_path):
    from patchfusion_b200.config import save_config
    with pytest.raises(ValueError):
        save_config({'model': {'x': float('nan')}}, str(tmp_path / 'c.py'))
    with pytest.raises(ValueError):
        save_config({'model': {'x': object()}}, str(tmp_path / 'd.py'))
