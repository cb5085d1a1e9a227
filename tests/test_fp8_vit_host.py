"""vit_precision = 'fp8_static' without a GPU: the config value and the ViT calibration table for vits / vitb / vitl, their
round trips, BaselinePretrain with the keys, a torch restatement of pf_layernorm_e4m3's rule, and the SASS of both
pf_gemm_pp_e4m3_kernel instantiations."""
import json
import math
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import fp8_vit_ref


def _cfg(enc='vits', **kw):
    from patchfusion_b200.configs import depth_anything_patchfusion
    cfg = depth_anything_patchfusion(enc, image_raw_shape=[1080, 1920], patch_split_num=[2, 2])
    cfg.update(kw)
    return cfg


def _table(enc='vits', v=2.0):
    from patchfusion_b200.params import vit_fp8_layers
    return {k: v + 0.25 * i for i, k in enumerate(vit_fp8_layers(_cfg(enc)))}


# ---------------------------------------------------------------------------------------------------- config
@pytest.mark.parametrize('enc,depth', [('vits', 12), ('vitb', 12), ('vitl', 24)])
def test_table_names(enc, depth):
    from patchfusion_b200.params import vit_fp8_layers
    names = vit_fp8_layers(_cfg(enc))
    assert len(names) == 6 * depth == len(set(names))
    assert names[:3] == ('coarse.0.qkv', 'coarse.0.fc1', 'coarse.0.fc2')
    assert names[-1] == 'fine.%d.fc2' % (depth - 1)
    assert {n.split('.')[0] for n in names} == {'coarse', 'fine'}


def test_vit_precision_values():
    from patchfusion_b200.model import PatchFusion
    from patchfusion_b200.params import vit_precision
    assert vit_precision(_cfg()) == 'bf16'
    for fp in ('bf16', 'fp8', 'fp8_static'):        # independent of fusion_precision: all six combinations build
        for vp in ('bf16', 'fp8_static'):
            m = PatchFusion(_cfg(fusion_precision=fp, vit_precision=vp))
            assert (m.fusion_precision, m.vit_precision) == (fp, vp)
    for bad in ('fp8', 'FP8_STATIC', 'e5m2', 'fp16', None):
        with pytest.raises(ValueError):
            PatchFusion(_cfg(vit_precision=bad))


@pytest.mark.parametrize('enc', ['vits', 'vitb', 'vitl'])
def test_table_validation(enc):
    from patchfusion_b200.model import PatchFusion
    from patchfusion_b200.params import vit_fp8_amax
    assert vit_fp8_amax(_cfg(enc)) is None
    good = _table(enc)
    assert vit_fp8_amax(_cfg(enc, vit_fp8_amax=good)) == good
    zero = dict(good, **{'fine.0.qkv': 0, 'coarse.3.fc2': np.float32(2.5)})
    assert vit_fp8_amax(_cfg(enc, vit_fp8_amax=zero))['fine.0.qkv'] == 0.0
    missing = dict(good)
    del missing['fine.5.fc1']
    depth = len(good) // 6
    bads = [missing, dict(good, extra=1.0), dict(good, **{'fine.%d.qkv' % depth: 1.0}),
            dict(good, **{'coarse.0.proj': 1.0}), dict(good, **{'fine.1.fc2': float('nan')}),
            dict(good, **{'fine.1.fc2': math.inf}), dict(good, **{'fine.1.fc2': -1e-3}),
            dict(good, **{'fine.1.fc2': '3.0'}), dict(good, **{'fine.1.fc2': None}), dict(good, **{'fine.1.fc2': True}),
            [1.0] * len(good), 'table']
    for bad in bads:
        with pytest.raises(ValueError):
            vit_fp8_amax(_cfg(enc, vit_fp8_amax=bad))
        for prec in ('fp8_static', 'bf16'):
            with pytest.raises(ValueError):
                PatchFusion(_cfg(enc, vit_precision=prec, vit_fp8_amax=bad))
    if enc != 'vitl':       # a vits / vitb table misses vitl's blocks 12-23
        with pytest.raises(ValueError):
            vit_fp8_amax(_cfg('vitl', vit_fp8_amax=good))


def test_without_table_builds_and_calibrate_refuses_bf16():
    from patchfusion_b200.model import PatchFusion
    m = PatchFusion(_cfg(vit_precision='fp8_static'))
    assert m.config.get('vit_fp8_amax') is None and callable(m.calibrate_fp8)
    with pytest.raises(ValueError, match='vit_precision'):
        PatchFusion(_cfg()).calibrate_fp8(None, None)


def test_table_round_trips(tmp_path):
    from patchfusion_b200.model import PatchFusion
    t = {k: float(np.float32(v) / np.float32(7.0)) for k, v in _table().items()}
    m = PatchFusion(_cfg(vit_precision='fp8_static', vit_fp8_amax=t))
    p = tmp_path / 'config.json'
    p.write_text(json.dumps(dict(m.config)))
    m2 = PatchFusion(json.loads(p.read_text()))
    assert m2.vit_precision == 'fp8_static' and dict(m2.config['vit_fp8_amax']) == t
    m.save_pretrained(str(tmp_path / 'hub'))
    m3 = PatchFusion.from_pretrained(str(tmp_path / 'hub'))
    assert m3.vit_precision == 'fp8_static' and dict(m3.config['vit_fp8_amax']) == t
    # config, not state: the state dict is the bf16 model's
    want = [(k, tuple(v.shape), v.dtype) for k, v in PatchFusion(_cfg()).state_dict().items()]
    assert [(k, tuple(v.shape), v.dtype) for k, v in m3.state_dict().items()] == want


def test_cfg_options():
    from patchfusion_b200.config import AttrDict, merge_options, parse_options
    cfg = AttrDict({'model': AttrDict({'config': AttrDict(_cfg())})})
    merge_options(cfg, parse_options(['model.config.vit_precision=fp8_static']))
    assert cfg['model']['config']['vit_precision'] == 'fp8_static'


def test_baseline_ignores_the_keys():
    from patchfusion_b200.baseline import BaselinePretrain
    from test_baseline_host import pretrain_model_cfg
    for target in ('coarse', 'fine'):
        cfg = pretrain_model_cfg('vits', target)
        cfg.pop('type')
        want = [(k, tuple(v.shape), v.dtype) for k, v in BaselinePretrain(**cfg).state_dict().items()]
        for table in (_table(), {'bogus': -1}, None):
            m = BaselinePretrain(**dict(cfg, vit_precision='fp8_static', vit_fp8_amax=table))
            assert [(k, tuple(v.shape), v.dtype) for k, v in m.state_dict().items()] == want


# ---------------------------------------------------------------------------------------------------- the LN rule
def test_layernorm_e4m3_rule_by_hand():
    """y = (x - mean) * rstd * w + b in fp32 with one fused multiply-add for the affine step, then e4m3_rn(sat(y * r))"""
    x = torch.tensor([[1.0, 2.0, 3.0, 4.0, -10.0, 0.0, 0.5, 1.5]])
    w = torch.tensor([1.0, -2.0, 0.5, 4.0, 1.0, 1.0, 64.0, 1.0])
    b = torch.tensor([0.0, 0.25, 0.0, -1.0, 0.0, 3.0, 0.0, 0.0])
    y = fp8_vit_ref.layernorm_f32(x, w, b, 1e-6)
    mean = x.double().mean()
    ref = (x.double() - mean) / torch.sqrt(((x.double() - mean) ** 2).mean() + 1e-6) * w.double() + b.double()
    assert (y.double() - ref).abs().max().item() < 1e-5
    q = fp8_vit_ref.layernorm_e4m3(x, w, b, 1e-6, 1.0)            # r = 448: past 1 saturates to 448
    assert q.dtype == torch.uint8
    f = q.view(fp8_vit_ref.E4M3).float()
    assert not torch.isnan(f).any() and f.abs().max().item() == 448.0
    import fp8_static_ref
    assert torch.equal(q, fp8_static_ref.quantize(y, 1.0).view(torch.uint8))


# ---------------------------------------------------------------------------------------------------- SASS
PP8_RE = re.compile(r'_ZN2pf22pf_gemm_pp_e4m3_kernelILb([01])EEEvNS_16GemmKernelParamsE')
PP_RE = re.compile(r'_ZN2pf17pf_gemm_pp_kernelILb([01])EEEvNS_16GemmKernelParamsE')
MMA_RE = re.compile(r'\b([HQ]GMMA)\.(\d+x\d+x\d+)\.')
LOCAL_RE = re.compile(r'\b(LDL|STL)\b')
ARRIVE_RE = re.compile(r'\bSYNCS\.ARRIVE\.TRANS64\.RED\b')
FENCE_RE = re.compile(r'\bMEMBAR\.ALL\.GPU\b')


@pytest.fixture(scope='module')
def sass_functions():
    from patchfusion_b200 import build
    path = build.build()
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    cuobjdump = os.path.join(os.path.dirname(nvcc), 'cuobjdump')
    sass = subprocess.run([cuobjdump, '-sass', path], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in sass.split('Function : ')[1:]:
        name, _, body = part.partition('\n')
        for tag, rx in (('e4m3', PP8_RE), ('bf16', PP_RE)):
            m = rx.match(name.strip())
            if m:
                funcs[(tag, int(m.group(1)))] = [l for l in body.split('\n') if re.search(r'/\*[0-9a-f]{4,}\*/', l)]
    return funcs


def test_instantiations(sass_functions):
    assert sorted(sass_functions) == [('bf16', 0), ('bf16', 1), ('e4m3', 0), ('e4m3', 1)]


@pytest.mark.parametrize('mc', [0, 1])
def test_e4m3_mainloop_sass(sass_functions, mc):
    """only QGMMA 64x128x32; a K block's eight MMAs (two 64-row halves x four k32 steps) back to back between warpgroup
    waits, with one group left in flight (DEPBAR.LE gsb0, 0x1)"""
    lines = sass_functions[('e4m3', mc)]
    shapes = [m.group(1) + ' ' + m.group(2) for m in (MMA_RE.search(l) for l in lines) if m]
    assert len(shapes) >= 8, len(shapes)
    assert set(shapes) == {'QGMMA 64x128x32'}, sorted(set(shapes))
    runs, n = [], 0
    for line in lines:
        if MMA_RE.search(line):
            n += 1
        elif 'WARPGROUP.DEPBAR' in line:
            if n:
                runs.append(n)
            n = 0
    assert runs and all(r == 8 for r in runs), runs
    assert any(re.search(r'WARPGROUP\.DEPBAR\.LE gsb0, 0x1 ;', l) for l in lines), 'no wait_group 1 in the mainloop'


@pytest.mark.parametrize('mc', [0, 1])
def test_e4m3_no_local_memory(sass_functions, mc):
    local = [l.strip() for l in sass_functions[('e4m3', mc)] if LOCAL_RE.search(l)]
    assert not local, local[:4]


def test_e4m3_remote_release_has_no_gpu_fence(sass_functions):
    lines = sass_functions[('e4m3', 1)]
    arrives = 0
    for i, line in enumerate(lines):
        if ARRIVE_RE.search(line):
            arrives += 1
            assert not any(FENCE_RE.search(l) for l in lines[max(0, i - 6):i]), lines[max(0, i - 6):i + 1]
    assert arrives > 0


def test_bf16_pp_kernel_has_no_fp8_mma(sass_functions):
    for mc in (0, 1):
        assert not any('QGMMA' in l for l in sass_functions[('bf16', mc)])
