"""dpt_precision = 'fp8_static' without a GPU: the config value and the DPT calibration table for vits / vitb / vitl, their
round trips, BaselinePretrain with the keys, a numpy model of the ReLU-copy staging layout of
pf_conv3_halo_e4m3_res_kernel, and the SASS of every instantiation of that kernel."""
import json
import math
import os
import re
import subprocess

import numpy as np
import pytest


def _cfg(enc='vits', **kw):
    from patchfusion_b200.configs import depth_anything_patchfusion
    cfg = depth_anything_patchfusion(enc, image_raw_shape=[1080, 1920], patch_split_num=[2, 2])
    cfg.update(kw)
    return cfg


def _table(enc='vits', v=2.0):
    from patchfusion_b200.params import dpt_fp8_layers
    return {k: v + 0.25 * i for i, k in enumerate(dpt_fp8_layers(_cfg(enc)))}


# ---------------------------------------------------------------------------------------------------- config
@pytest.mark.parametrize('enc', ['vits', 'vitb', 'vitl'])
def test_table_names(enc):
    from patchfusion_b200.params import DPT_FP8_CONVS, dpt_fp8_layers
    names = dpt_fp8_layers(_cfg(enc))
    assert len(names) == 38 == len(set(names)) and len(DPT_FP8_CONVS) == 19
    per = {'%s.layer%d_rn' % (b, i) for b in ('coarse', 'fine') for i in range(1, 5)}
    per |= {'%s.refinenet%d.resConfUnit%d.conv%d' % (b, i, u, k) for b in ('coarse', 'fine') for i in (1, 2, 3)
            for u in (1, 2) for k in (1, 2)}
    per |= {'%s.refinenet4.resConfUnit2.conv%d' % (b, k) for b in ('coarse', 'fine') for k in (1, 2)}
    per |= {'%s.output_conv1' % b for b in ('coarse', 'fine')}
    assert set(names) == per
    # the names are the state dict's: every one is a 3x3 conv of its branch's depth head
    from patchfusion_b200.model import PatchFusion
    sd = PatchFusion(_cfg(enc)).state_dict()
    for n in names:
        b, conv = n.split('.', 1)
        w = sd['%s_branch.core.core.depth_head.scratch.%s.weight' % (b, conv)]
        assert tuple(w.shape[2:]) == (3, 3), n


def test_dpt_precision_values():
    from patchfusion_b200.model import PatchFusion
    from patchfusion_b200.params import dpt_precision
    assert dpt_precision(_cfg()) == 'bf16'
    for dp in ('bf16', 'fp8_static'):       # independent of the other two keys
        for vp in ('bf16', 'fp8_static'):
            for fp in ('bf16', 'fp8', 'fp8_static'):
                m = PatchFusion(_cfg(fusion_precision=fp, vit_precision=vp, dpt_precision=dp))
                assert (m.fusion_precision, m.vit_precision, m.dpt_precision) == (fp, vp, dp)
    for bad in ('fp8', 'FP8_STATIC', 'e5m2', 'fp16', None):
        with pytest.raises(ValueError):
            PatchFusion(_cfg(dpt_precision=bad))


@pytest.mark.parametrize('enc', ['vits', 'vitb', 'vitl'])
def test_table_validation(enc):
    from patchfusion_b200.model import PatchFusion
    from patchfusion_b200.params import dpt_fp8_amax
    assert dpt_fp8_amax(_cfg(enc)) is None
    good = _table(enc)
    assert dpt_fp8_amax(_cfg(enc, dpt_fp8_amax=good)) == good
    zero = dict(good, **{'fine.layer1_rn': 0, 'coarse.output_conv1': np.float32(2.5)})
    assert dpt_fp8_amax(_cfg(enc, dpt_fp8_amax=zero))['fine.layer1_rn'] == 0.0
    missing = dict(good)
    del missing['fine.refinenet2.resConfUnit1.conv2']
    bads = [missing, dict(good, extra=1.0), dict(good, **{'fine.refinenet4.resConfUnit1.conv1': 1.0}),
            dict(good, **{'coarse.output_conv2.0': 1.0}), dict(good, **{'fine.layer2_rn': float('nan')}),
            dict(good, **{'fine.layer2_rn': math.inf}), dict(good, **{'fine.layer2_rn': -1e-3}),
            dict(good, **{'fine.layer2_rn': '3.0'}), dict(good, **{'fine.layer2_rn': None}),
            dict(good, **{'fine.layer2_rn': True}), [1.0] * len(good), 'table']
    for bad in bads:
        with pytest.raises(ValueError):
            dpt_fp8_amax(_cfg(enc, dpt_fp8_amax=bad))
        for prec in ('fp8_static', 'bf16'):
            with pytest.raises(ValueError):
                PatchFusion(_cfg(enc, dpt_precision=prec, dpt_fp8_amax=bad))


def test_without_table_builds_and_calibrate_refuses_bf16():
    from patchfusion_b200.model import PatchFusion
    m = PatchFusion(_cfg(dpt_precision='fp8_static'))
    assert m.config.get('dpt_fp8_amax') is None and callable(m.calibrate_fp8)
    with pytest.raises(ValueError, match='vit_precision'):
        PatchFusion(_cfg()).calibrate_fp8(None, None)
    with pytest.raises(ValueError, match='dpt_precision'):
        PatchFusion(_cfg()).calibrate_fp8(None, None)


def test_table_round_trips(tmp_path):
    from patchfusion_b200.model import PatchFusion
    t = {k: float(np.float32(v) / np.float32(7.0)) for k, v in _table().items()}
    m = PatchFusion(_cfg(dpt_precision='fp8_static', dpt_fp8_amax=t))
    p = tmp_path / 'config.json'
    p.write_text(json.dumps(dict(m.config)))
    m2 = PatchFusion(json.loads(p.read_text()))
    assert m2.dpt_precision == 'fp8_static' and dict(m2.config['dpt_fp8_amax']) == t
    m.save_pretrained(str(tmp_path / 'hub'))
    m3 = PatchFusion.from_pretrained(str(tmp_path / 'hub'))
    assert m3.dpt_precision == 'fp8_static' and dict(m3.config['dpt_fp8_amax']) == t
    # config, not state: the state dict is the bf16 model's
    want = [(k, tuple(v.shape), v.dtype) for k, v in PatchFusion(_cfg()).state_dict().items()]
    assert [(k, tuple(v.shape), v.dtype) for k, v in m3.state_dict().items()] == want


def test_cfg_options():
    from patchfusion_b200.config import AttrDict, merge_options, parse_options
    cfg = AttrDict({'model': AttrDict({'config': AttrDict(_cfg())})})
    merge_options(cfg, parse_options(['model.config.dpt_precision=fp8_static']))
    assert cfg['model']['config']['dpt_precision'] == 'fp8_static'


def test_baseline_ignores_the_keys():
    from patchfusion_b200.baseline import BaselinePretrain
    from test_baseline_host import pretrain_model_cfg
    for target in ('coarse', 'fine'):
        cfg = pretrain_model_cfg('vits', target)
        cfg.pop('type')
        want = [(k, tuple(v.shape), v.dtype) for k, v in BaselinePretrain(**cfg).state_dict().items()]
        for table in (_table(), {'bogus': -1}, None):
            m = BaselinePretrain(**dict(cfg, dpt_precision='fp8_static', dpt_fp8_amax=table))
            assert [(k, tuple(v.shape), v.dtype) for k, v in m.state_dict().items()] == want


# ---------------------------------------------------------------------------------------------------- copy layout
def _copy_offsets():
    """csrc/pf_gemm.cu epilogue_tile_tma_res, the e4m3 ReLU copy: (lane, h, j) -> the two byte offsets its e4m3x2
    lands at in the 16 x 64-byte staging tile, and the (row, column) pairs they hold.  Row lane / 4 is pixel (2 warp,
    lane / 4) of the 16 x 8 pixel tile, row lane / 4 + 8 the pixel below it: the {64 B, 8 px, 2 rows} box order."""
    out = {}
    for lane in range(32):
        r0, q = lane >> 2, lane & 3
        swz8 = (r0 >> 1) & 3
        for h in range(2):
            for j in range(4):
                b = 32 * h + 8 * j + 2 * q
                off = (((b >> 4) ^ swz8) << 4) | (b & 15)
                out[(lane, h, j)] = [(r0 * 64 + off, r0, b), ((r0 + 8) * 64 + off, r0 + 8, b)]
    return out


def test_relu_copy_staging_layout_model():
    """every byte of the staging tile is written exactly once, at the place SWIZZLE_64B expects its (row, column)
    (16-byte piece j of row r at j ^ ((r >> 1) & 3)), and each store instruction's 32 lanes fall in distinct banks"""
    offs = _copy_offsets()
    written = np.zeros(16 * 64, dtype=np.int32)
    for lst in offs.values():
        for off, r, b in lst:
            for e in range(2):
                written[off + e] += 1
                col = b + e
                assert off + e == r * 64 + (((col >> 4) ^ ((r >> 1) & 3)) << 4) + (col & 15)
    assert (written == 1).all()
    for h in range(2):
        for j in range(4):
            for which in range(2):
                words = {}
                for lane in range(32):
                    off = offs[(lane, h, j)][which][0]
                    words.setdefault((off >> 2) & 31, set()).add(off >> 2)
                # lanes sharing a bank share its 32-bit word (the two halves of one word): no conflict
                assert all(len(w) == 1 for w in words.values()), (h, j, which)
                # eight rows per instruction, each in its own group of four banks
                groups = {((offs[(lane, h, j)][which][0] >> 2) & 31) >> 2 for lane in range(32)}
                assert len(groups) == 8, (h, j, which, groups)


# ---------------------------------------------------------------------------------------------------- SASS
RES_RE = re.compile(r'_ZN2pf29pf_conv3_halo_e4m3_res_kernelILi(\d)ELi(\d+)EEEvNS_16GemmKernelParamsE')
QGMMA_RE = re.compile(r'\bQGMMA\.(\d+x\d+x\d+)\.F32\.E4M3\.E4M3\b')
ANY_GMMA_RE = re.compile(r'\b[HQ]GMMA\.')
LOCAL_RE = re.compile(r'\b(LDL|STL)\b')
ARRIVE_RE = re.compile(r'\bSYNCS\.ARRIVE\.TRANS64\.RED\b')
FENCE_RE = re.compile(r'\bMEMBAR\.ALL\.GPU\b')


@pytest.fixture(scope='module')
def res_functions():
    from patchfusion_b200 import build
    path = build.build()
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    cuobjdump = os.path.join(os.path.dirname(nvcc), 'cuobjdump')
    sass = subprocess.run([cuobjdump, '-sass', path], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in sass.split('Function : ')[1:]:
        name, _, body = part.partition('\n')
        m = RES_RE.match(name.strip())
        if m:
            funcs[(int(m.group(1)), int(m.group(2)))] = [l for l in body.split('\n') if re.search(r'/\*[0-9a-f]{4,}\*/', l)]
    return funcs


def test_res_instantiations(res_functions):
    assert sorted(res_functions) == [(cl, bn) for cl in (1, 2, 4) for bn in (64, 128)]


@pytest.mark.parametrize('cl', [1, 2, 4])
@pytest.mark.parametrize('bn', [64, 128])
def test_res_mainloop_sass(res_functions, cl, bn):
    lines = res_functions[(cl, bn)]
    body = '\n'.join(lines)
    shapes = QGMMA_RE.findall(body)
    assert len(shapes) >= 18, len(shapes)
    assert set(shapes) == {'64x%dx32' % bn}, sorted(set(shapes))
    assert len(shapes) == len(ANY_GMMA_RE.findall(body)), 'an MMA that is not 64xBNx32 E4M3'
    assert re.search(r'WARPGROUP\.DEPBAR\.LE gsb0, 0x1 ;', body), 'no wait_group 1 in the mainloop'
    # no local memory between the first and the last QGMMA of a chunk (BN = 128 spills a few epilogue values, DESIGN.md
    # section 3; the mainloop must not touch them)
    mma = [i for i, l in enumerate(lines) if QGMMA_RE.search(l)]
    assert not [l for l in lines[mma[0]:mma[-1] + 1] if LOCAL_RE.search(l)], 'local memory in the mainloop'
    if bn == 64:
        assert not [l for l in lines if LOCAL_RE.search(l)], 'local memory in the kernel'
    # the epilogue: stmatrix staging, e4m3x2 conversions of the ReLU copy, bulk tensor stores
    assert re.search(r'\bSTSM\b', body), 'no stmatrix'
    assert re.search(r'\bF2FP\.SATFINITE\.E4M3\.F32\.PACK_AB', body), 'no e4m3x2 conversion'
    assert 'UTMASTG' in body


@pytest.mark.parametrize('cl', [2, 4])
@pytest.mark.parametrize('bn', [64, 128])
def test_res_stage_release_without_gpu_fence(res_functions, cl, bn):
    lines = res_functions[(cl, bn)]
    arrives = [i for i, l in enumerate(lines) if ARRIVE_RE.search(l)]
    assert arrives, 'no remote arrive in a multicast instantiation'
    assert not [i for i in arrives if any(FENCE_RE.search(l) for l in lines[max(0, i - 6):i])], \
        'MEMBAR.ALL.GPU in front of a remote stage release'
