"""fusion_precision = 'fp8_static' without a GPU: the config value and the calibration table, their round trips, the
saturating static rule by hand, a numpy model of the e4m3 output epilogue's staging layout, and the SASS of every
static-scale E4M3 halo conv instantiation."""
import json
import math
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import fp8_static_ref


def _cfg(**kw):
    from patchfusion_b200.configs import depth_anything_patchfusion
    cfg = depth_anything_patchfusion('vits', image_raw_shape=[1080, 1920], patch_split_num=[2, 2])
    cfg.update(kw)
    return cfg


def _table(v=3.0):
    from patchfusion_b200.params import FP8_LAYERS
    return {k: v + i for i, k in enumerate(FP8_LAYERS)}


# ---------------------------------------------------------------------------------------------------- config
def test_fp8_layers_are_the_34_unet_convs():
    from patchfusion_b200.params import FP8_LAYERS
    assert len(FP8_LAYERS) == 34 == len(set(FP8_LAYERS))
    assert {n.rsplit('.', 1)[0] for n in FP8_LAYERS} == (
        {'inc'} | {'down%d' % i for i in range(5)} | {'up%d' % i for i in range(1, 6)} | {'cv%d' % i for i in range(6)})


def test_fp8_static_value_accepted():
    from patchfusion_b200.model import PatchFusion
    from patchfusion_b200.params import fusion_precision
    assert fusion_precision(_cfg(fusion_precision='fp8_static')) == 'fp8_static'
    assert PatchFusion(_cfg(fusion_precision='fp8_static')).fusion_precision == 'fp8_static'
    m = PatchFusion(_cfg(fusion_precision='fp8_static', fusion_fp8_amax=_table()))
    assert m.config['fusion_fp8_amax']['cv5.1'] == _table()['cv5.1']
    for bad in ('fp8-static', 'FP8_STATIC', 'static', 'e5m2'):
        with pytest.raises(ValueError):
            PatchFusion(_cfg(fusion_precision=bad))


def test_table_validation():
    from patchfusion_b200.model import PatchFusion
    from patchfusion_b200.params import fusion_fp8_amax
    assert fusion_fp8_amax(_cfg()) is None
    good = _table()
    assert fusion_fp8_amax(_cfg(fusion_fp8_amax=good)) == good
    zero = dict(good, **{'inc.0': 0, 'down3.1': np.float32(2.5)})
    assert fusion_fp8_amax(_cfg(fusion_fp8_amax=zero))['inc.0'] == 0.0
    missing = dict(good)
    del missing['up3.0']
    bads = [missing, dict(good, extra=1.0), dict(good, **{'inc.2': 1.0}),
            dict(good, **{'cv0.0': float('nan')}), dict(good, **{'cv0.0': math.inf}), dict(good, **{'cv0.0': -1e-3}),
            dict(good, **{'cv0.0': '3.0'}), dict(good, **{'cv0.0': None}), dict(good, **{'cv0.0': True}),
            [1.0] * 34, 'table']
    for bad in bads:
        with pytest.raises(ValueError):
            fusion_fp8_amax(_cfg(fusion_fp8_amax=bad))
        for prec in ('fp8_static', 'fp8', 'bf16'):
            with pytest.raises(ValueError):
                PatchFusion(_cfg(fusion_precision=prec, fusion_fp8_amax=bad))


def test_fp8_static_without_table_builds():
    """the model builds (and can be calibrated); its forward refuses, on the GPU (tests/test_gpu_fp8_static.py)"""
    from patchfusion_b200.model import PatchFusion
    m = PatchFusion(_cfg(fusion_precision='fp8_static'))
    assert m.config.get('fusion_fp8_amax') is None
    assert callable(m.calibrate_fp8)


def test_calibrate_refuses_bf16_models():
    from patchfusion_b200.model import PatchFusion
    with pytest.raises(ValueError):
        PatchFusion(_cfg()).calibrate_fp8(None, None)


def test_table_round_trips(tmp_path):
    from patchfusion_b200.model import PatchFusion
    t = {k: float(np.float32(v) / np.float32(7.0)) for k, v in _table().items()}    # float32 values, as calibrated
    m = PatchFusion(_cfg(fusion_precision='fp8_static', fusion_fp8_amax=t))
    p = tmp_path / 'config.json'
    p.write_text(json.dumps(dict(m.config)))
    m2 = PatchFusion(json.loads(p.read_text()))
    assert m2.fusion_precision == 'fp8_static' and dict(m2.config['fusion_fp8_amax']) == t
    m.save_pretrained(str(tmp_path / 'hub'))
    m3 = PatchFusion.from_pretrained(str(tmp_path / 'hub'))
    assert m3.fusion_precision == 'fp8_static' and dict(m3.config['fusion_fp8_amax']) == t
    # the table is config, not state: the state-dict layout is the bf16 model's
    assert list(m3.state_dict()) == list(PatchFusion(_cfg()).state_dict())


def test_cfg_options():
    from patchfusion_b200.config import AttrDict, merge_options, parse_options
    cfg = AttrDict({'model': AttrDict({'config': AttrDict(_cfg())})})
    merge_options(cfg, parse_options(['model.config.fusion_precision=fp8_static']))
    assert cfg['model']['config']['fusion_precision'] == 'fp8_static'


def test_baseline_ignores_the_table():
    from patchfusion_b200.baseline import BaselinePretrain
    from test_baseline_host import pretrain_model_cfg
    for target in ('coarse', 'fine'):
        cfg = pretrain_model_cfg('vits', target)
        cfg.pop('type')
        want = [(k, tuple(v.shape), v.dtype) for k, v in BaselinePretrain(**cfg).state_dict().items()]
        for table in (_table(), {'bogus': -1}, None):
            m = BaselinePretrain(**dict(cfg, fusion_precision='fp8_static', fusion_fp8_amax=table))
            assert [(k, tuple(v.shape), v.dtype) for k, v in m.state_dict().items()] == want


# ---------------------------------------------------------------------------------------------------- the rule
def test_static_rule_by_hand():
    from patchfusion_b200 import ops
    # amax 7: r = 64 exactly; values past the amax saturate at 448, never NaN; -0 keeps its sign
    v = torch.tensor([0.0, -0.0, 1.0, -3.5, 7.0, 7.1, 7.25, 8.0, -100.0, 1e30, float('inf'), -float('inf')])
    q = fp8_static_ref.quantize(v, 7.0)
    assert q.float()[:8].tolist() == [0.0, -0.0, 64.0, -224.0, 448.0, 448.0, 448.0, 448.0]
    assert q.float()[8:].tolist() == [-448.0, 448.0, 448.0, -448.0]
    assert q.view(torch.uint8)[1].item() == 0x80
    # just above 448 after scaling: 7.1 * 64 = 454.4 and 7.25 * 64 = 464 round to 448; 7.5 * 64 = 480 is past what
    # torch's unclamped cast keeps finite (it gives NaN), the saturating rule gives 448
    assert torch.isnan((torch.tensor([7.5]) * 64).to(fp8_static_ref.E4M3).float()).all()
    assert fp8_static_ref.quantize(torch.tensor([7.5]), 7.0).float().item() == 448.0
    assert not torch.isnan(q.float()).any()
    # NaN stays NaN; amax 0 gives r = 0: every finite value quantizes to zero
    assert torch.isnan(fp8_static_ref.quantize(torch.tensor([float('nan')]), 1.0).float()).all()
    assert (fp8_static_ref.quantize(torch.tensor([3.0, -2.0]), 0.0).float() == 0).all()
    # the host's fp32 ratio / scale equal the one-division rule
    for a in (7.0, 0.3, 1e-20, 3.4e38, 0.0):
        assert ops.e4m3_static_ratio(a) == float(fp8_static_ref.ratio(a))
        assert ops.e4m3_static_scale(a) == float(fp8_static_ref.scale(a))


def test_static_map_layout():
    g = torch.Generator().manual_seed(0)
    a = torch.randn(2, 3, 4, 8, generator=g).bfloat16()
    b = torch.randn(2, 3, 4, 72, generator=g).bfloat16() * 30
    q = fp8_static_ref.quantize_static_ref([a, b], [5, 70], 4.0)
    assert q.shape == (2, 3, 4, 64 + 128)
    assert (q[..., 5:64] == 0).all() and (q[..., 64 + 70:] == 0).all()
    assert torch.equal(q[..., 64:64 + 70], fp8_static_ref.quantize(b[..., :70].float(), 4.0).view(torch.uint8))


# ---------------------------------------------------------------------------------------------------- epilogue layout
def _staging_offsets():
    """csrc/pf_gemm.cu epilogue_tile_tma_e4m3: (lane, h, j) -> the two byte offsets its e4m3x2 lands at, and the
    (row, column) pairs they hold"""
    out = {}
    for lane in range(32):
        r0, q = lane >> 2, lane & 3
        swz = (r0 >> 1) & 3
        for h in range(2):
            for j in range(4):
                b = 32 * h + 8 * j + 2 * q
                off = (((b >> 4) ^ swz) << 4) | (b & 15)
                out[(lane, h, j)] = [(r0 * 64 + off, r0, b), ((r0 + 8) * 64 + off, r0 + 8, b)]
    return out


def test_e4m3_epilogue_layout_model():
    """every byte of the 16 x 64 staging tile is written exactly once, at the place SWIZZLE_64B expects its (row,
    column) (16-byte piece j of row r at j ^ ((r >> 1) & 3)), and no store instruction has a bank conflict"""
    offs = _staging_offsets()
    written = np.zeros(16 * 64, dtype=np.int32)
    for lst in offs.values():
        for off, r, b in lst:
            for e in range(2):          # the two bytes of the e4m3x2: columns b, b + 1
                written[off + e] += 1
                col = b + e
                want = r * 64 + (((col >> 4) ^ ((r >> 1) & 3)) << 4) + (col & 15)
                assert off + e == want
    assert (written == 1).all()
    for h in range(2):
        for j in range(4):
            for which in range(2):      # the row lane / 4 store, then the row lane / 4 + 8 store
                banks = {}
                for lane in range(32):
                    off = offs[(lane, h, j)][which][0]
                    banks.setdefault((off >> 2) & 31, set()).add(off >> 2)
                assert all(len(words) == 1 for words in banks.values()), (h, j, which)


# ---------------------------------------------------------------------------------------------------- SASS
Q8_RE = re.compile(r'_ZN2pf28pf_conv3_halo_e4m3_q8_kernelILi(\d)ELi(\d+)EEEvNS_16GemmKernelParamsE')
QGMMA_RE = re.compile(r'\bQGMMA\.(\d+x\d+x\d+)\.F32\.E4M3\.E4M3\b')
ANY_GMMA_RE = re.compile(r'\b[HQ]GMMA\.')
LOCAL_RE = re.compile(r'\b(LDL|STL)\b')
ARRIVE_RE = re.compile(r'\bSYNCS\.ARRIVE\.TRANS64\.RED\b')
FENCE_RE = re.compile(r'\bMEMBAR\.ALL\.GPU\b')


@pytest.fixture(scope='module')
def q8_functions():
    from patchfusion_b200 import build
    path = build.build()
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    cuobjdump = os.path.join(os.path.dirname(nvcc), 'cuobjdump')
    sass = subprocess.run([cuobjdump, '-sass', path], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in sass.split('Function : ')[1:]:
        name, _, body = part.partition('\n')
        m = Q8_RE.match(name.strip())
        if m:
            funcs[(int(m.group(1)), int(m.group(2)))] = [l for l in body.split('\n') if re.search(r'/\*[0-9a-f]{4,}\*/', l)]
    return funcs


def test_q8_instantiations(q8_functions):
    assert sorted(q8_functions) == [(cl, bn) for cl in (1, 2, 4) for bn in (32, 64, 128, 192)]


@pytest.mark.parametrize('cl', [1, 2, 4])
@pytest.mark.parametrize('bn', [32, 64, 128, 192])
def test_q8_mainloop_sass(q8_functions, cl, bn):
    lines = q8_functions[(cl, bn)]
    body = '\n'.join(lines)
    shapes = QGMMA_RE.findall(body)
    assert len(shapes) >= 18, len(shapes)
    assert set(shapes) == {'64x%dx32' % bn}, sorted(set(shapes))
    assert len(shapes) == len(ANY_GMMA_RE.findall(body)), 'an MMA that is not 64xBNx32 E4M3'
    assert re.search(r'WARPGROUP\.DEPBAR\.LE gsb0, 0x1 ;', body), 'no wait_group 1 in the mainloop'
    assert not [l for l in lines if LOCAL_RE.search(l)], 'local memory in the kernel'
    # the e4m3 output: saturating conversions and bulk tensor stores
    assert re.search(r'\bF2FP\.SATFINITE\.E4M3\.F32\.PACK_AB', body), 'no e4m3x2 conversion'
    assert 'UTMASTG' in body


@pytest.mark.parametrize('cl', [2, 4])
@pytest.mark.parametrize('bn', [32, 64, 128, 192])
def test_q8_stage_release_without_gpu_fence(q8_functions, cl, bn):
    lines = q8_functions[(cl, bn)]
    arrives = [i for i, l in enumerate(lines) if ARRIVE_RE.search(l)]
    assert arrives, 'no remote arrive in a multicast instantiation'
    assert not [i for i in arrives if any(FENCE_RE.search(l) for l in lines[max(0, i - 6):i])], \
        'MEMBAR.ALL.GPU in front of a remote stage release'


def test_existing_kernel_symbols_kept():
    from patchfusion_b200 import build
    path = build.build()
    out = subprocess.check_output(['nm', '-C', path], text=True)
    for cl in (1, 2, 4):
        for bn in (32, 64, 128, 192):
            assert 'pf::pf_conv3_halo_kernel<%d, %d>' % (cl, bn) in out
            assert 'pf::pf_conv3_halo_e4m3_kernel<%d, %d>' % (cl, bn) in out
            assert 'pf::pf_conv3_halo_e4m3_q8_kernel<%d, %d>' % (cl, bn) in out
    assert 'pf_quantize_e4m3_static' in out and 'pf_quantize_e4m3_tiles' in out
