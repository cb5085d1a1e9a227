"""fusion_precision = 'fp8' without a GPU: the config key, the SASS of the E4M3 halo conv, the torch emulation of the
quantizers against hand-worked values, and the quantization cost of the FP8 U-Net on the vits_case0 fixture (the
FP8-emulating oracle against the fp32 oracle, reported, not asserted: it measures synthetic weights)."""
import json
import os
import re
import subprocess

import pytest
import torch

import fp8_ref

GOLD = os.path.join(os.path.dirname(__file__), 'golden')


# ---------------------------------------------------------------------------------------------------- config
def _cfg(**kw):
    from patchfusion_b200.configs import depth_anything_patchfusion
    cfg = depth_anything_patchfusion('vits', image_raw_shape=[1080, 1920], patch_split_num=[2, 2])
    cfg.update(kw)
    return cfg


def test_fusion_precision_default_and_values():
    from patchfusion_b200.model import PatchFusion
    from patchfusion_b200.params import fusion_precision
    assert fusion_precision(_cfg()) == 'bf16'
    assert PatchFusion(_cfg()).fusion_precision == 'bf16'
    assert PatchFusion(_cfg(fusion_precision='fp8')).fusion_precision == 'fp8'
    for bad in ('fp16', 'FP8', 'e4m3', None, 8):
        with pytest.raises(ValueError):
            PatchFusion(_cfg(fusion_precision=bad))


def test_fusion_precision_survives_save_and_load(tmp_path):
    from patchfusion_b200.model import PatchFusion
    m = PatchFusion(_cfg(fusion_precision='fp8'))
    p = tmp_path / 'config.json'
    p.write_text(json.dumps(dict(m.config)))
    m2 = PatchFusion(json.loads(p.read_text()))
    assert m2.config['fusion_precision'] == 'fp8' and m2.fusion_precision == 'fp8'
    if hasattr(m, 'save_pretrained') and hasattr(PatchFusion, 'from_pretrained'):
        try:
            m.save_pretrained(str(tmp_path / 'hub'))
        except (ImportError, NotImplementedError):
            return
        m3 = PatchFusion.from_pretrained(str(tmp_path / 'hub'))
        assert m3.fusion_precision == 'fp8'


def test_fusion_precision_cfg_option():
    from patchfusion_b200.config import AttrDict, merge_options, parse_options
    cfg = AttrDict({'model': AttrDict({'config': AttrDict(_cfg())})})
    merge_options(cfg, parse_options(['model.config.fusion_precision=fp8']))
    assert cfg['model']['config']['fusion_precision'] == 'fp8'


def test_baseline_ignores_fusion_precision():
    """BaselinePretrain has no fusion stage: a model dict carrying the key, with any value, builds the same model"""
    from patchfusion_b200.baseline import BaselinePretrain
    from test_baseline_host import pretrain_model_cfg
    for target in ('coarse', 'fine'):
        cfg = pretrain_model_cfg('vits', target)
        cfg.pop('type')
        want = [(k, tuple(v.shape), v.dtype) for k, v in BaselinePretrain(**cfg).state_dict().items()]
        for value in ('fp8', 'bf16', 'bogus'):
            m = BaselinePretrain(**dict(cfg, fusion_precision=value))
            assert [(k, tuple(v.shape), v.dtype) for k, v in m.state_dict().items()] == want
            assert m.branch == target


# ---------------------------------------------------------------------------------------------------- SASS
E4M3_RE = re.compile(r'_ZN2pf25pf_conv3_halo_e4m3_kernelILi(\d)ELi(\d+)EEEvNS_16GemmKernelParamsE')
HGMMA_RE = re.compile(r'\bQGMMA\.(\d+x\d+x\d+)\.F32\.E4M3\.E4M3\b')     # FP8 wgmma disassembles as QGMMA
ANY_HGMMA_RE = re.compile(r'\b[HQ]GMMA\.')
LOCAL_RE = re.compile(r'\b(LDL|STL)\b')
ARRIVE_RE = re.compile(r'\bSYNCS\.ARRIVE\.TRANS64\.RED\b')
FENCE_RE = re.compile(r'\bMEMBAR\.ALL\.GPU\b')


@pytest.fixture(scope='module')
def e4m3_functions():
    from patchfusion_b200 import build
    path = build.build()
    nvcc = os.environ.get('NVCC', '/usr/local/cuda/bin/nvcc')
    cuobjdump = os.path.join(os.path.dirname(nvcc), 'cuobjdump')
    sass = subprocess.run([cuobjdump, '-sass', path], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for part in sass.split('Function : ')[1:]:
        name, _, body = part.partition('\n')
        m = E4M3_RE.match(name.strip())
        if m:
            funcs[(int(m.group(1)), int(m.group(2)))] = [l for l in body.split('\n') if re.search(r'/\*[0-9a-f]{4,}\*/', l)]
    return funcs


def test_e4m3_instantiations(e4m3_functions):
    assert sorted(e4m3_functions) == [(cl, bn) for cl in (1, 2, 4) for bn in (32, 64, 128, 192)]


@pytest.mark.parametrize('cl', [1, 2, 4])
@pytest.mark.parametrize('bn', [32, 64, 128, 192])
def test_e4m3_mainloop_sass(e4m3_functions, cl, bn):
    lines = e4m3_functions[(cl, bn)]
    body = '\n'.join(lines)
    shapes = HGMMA_RE.findall(body)
    # nine taps x two k32 steps per 64-channel chunk, fully unrolled, every one an E4M3 x E4M3 MMA
    assert len(shapes) >= 18, len(shapes)
    assert set(shapes) == {'64x%dx32' % bn}, sorted(set(shapes))
    assert len(shapes) == len(ANY_HGMMA_RE.findall(body)), 'an HGMMA that is not 64xBNx32 E4M3'
    # the two k32 steps of a tap go out back to back
    runs, n = [], 0
    for line in lines:
        if ANY_HGMMA_RE.search(line):
            n += 1
        elif 'WARPGROUP.DEPBAR' in line:
            if n:
                runs.append(n)
            n = 0
    assert runs and min(runs) >= 2 and all(r % 2 == 0 for r in runs), runs
    # one tap's group stays in flight
    assert re.search(r'WARPGROUP\.DEPBAR\.LE gsb0, 0x1 ;', body), 'no wait_group 1 in the mainloop'
    # no local memory between the first and the last HGMMA of the mainloop
    idx = [i for i, l in enumerate(lines) if ANY_HGMMA_RE.search(l)]
    assert not [l for l in lines[idx[0]:idx[-1] + 1] if LOCAL_RE.search(l)], 'local memory inside the mainloop'
    assert not [l for l in lines if LOCAL_RE.search(l)], 'local memory in the kernel'


@pytest.mark.parametrize('cl', [2, 4])
@pytest.mark.parametrize('bn', [32, 64, 128, 192])
def test_e4m3_stage_release_without_gpu_fence(e4m3_functions, cl, bn):
    """the multicast stages are released to the peer CTAs with plain remote arrives (tests/test_stage_release_sass.py)"""
    lines = e4m3_functions[(cl, bn)]
    arrives = [i for i, l in enumerate(lines) if ARRIVE_RE.search(l)]
    assert arrives, 'no remote arrive in a multicast instantiation'
    assert not [i for i in arrives if any(FENCE_RE.search(l) for l in lines[max(0, i - 6):i])], \
        'MEMBAR.ALL.GPU in front of a remote stage release'


def test_bf16_halo_kernel_names_unchanged():
    """the bf16 instantiations keep their symbols: the FP8 path is a separate kernel"""
    from patchfusion_b200 import build
    path = build.build()
    out = subprocess.check_output(['nm', '-C', path], text=True)
    for cl in (1, 2, 4):
        for bn in (32, 64, 128, 192):
            assert 'pf::pf_conv3_halo_kernel<%d, %d>' % (cl, bn) in out
            assert 'pf::pf_conv3_halo_e4m3_kernel<%d, %d>' % (cl, bn) in out


# ---------------------------------------------------------------------------------------------------- emulation
def test_quantize_rule_by_hand():
    v = torch.tensor([[0.0, -0.0, 1.0, -3.5, 7.0], [0.0, 0.0, -0.0, 0.0, 0.0], [1e-6, 2.0, 0.0, 0.0, -448.0]])
    q, s = fp8_ref.quantize(v, fp8_ref.group_amax(v))
    assert s.tolist() == [7.0 / 448, 0.0, 1.0]
    # 448 / 7 = 64: exact; -0.0 keeps its sign; an all-zero group is zeros with scale 0
    assert q[0].float().tolist() == [0.0, -0.0, 64.0, -224.0, 448.0]
    assert q.view(torch.uint8)[0, 1].item() == 0x80
    assert (q[1].float() == 0).all()
    # 1e-6 * 1 is below half the smallest e4m3 subnormal (2^-9): rounds to zero
    assert q[2].float().tolist() == [0.0, 2.0, 0.0, 0.0, -448.0]
    nan = fp8_ref.group_amax(torch.tensor([[1.0, float('nan'), 2.0]]))
    assert torch.isnan(nan).all()


def test_pack_and_quantize_ref_layout():
    g = torch.Generator().manual_seed(0)
    w = torch.randn(40, 5 + 70, 3, 3, generator=g)
    panel, s_w = fp8_ref.pack_weight_e4m3_ref(w, [5, 70], n_pad=64)
    assert panel.shape == (64, 9 * 64 + 9 * 128) and s_w.shape == (40,)
    assert (panel[40:] == 0).all()
    # tap 4 (the centre) of source 1, channel 3 of row 7
    q = (w * (448 / w.flatten(1).abs().amax(1)).view(-1, 1, 1, 1)).to(fp8_ref.E4M3).view(torch.uint8)
    assert panel[7, 9 * 64 + 4 * 128 + 3] == q[7, 5 + 3, 1, 1]
    assert (panel[:, 9 * 64 + 4 * 128 + 70:9 * 64 + 5 * 128] == 0).all()
    x = torch.randn(3, 4, 5, 8, generator=g).bfloat16()
    qm, s_a = fp8_ref.quantize_tiles_ref([x], [5])
    assert qm.shape == (3, 4, 5, 64) and (qm[..., 5:] == 0).all()
    assert torch.equal(s_a, x[..., :5].float().flatten(1).abs().amax(1) / 448)


@pytest.mark.timeout(1800)
def test_fp8_emulation_cost_on_vits_case0():
    """The FP8 U-Net's distance from the fp32 oracle on the fixture's two fine tiles (quantization cost on synthetic
    weights: printed, not asserted)"""
    from oracle import pf_oracle as po
    from oracle.make_golden import case_inputs
    case = json.load(open(os.path.join(GOLD, 'vits_case0.json')))
    cfg, sd, img = case_inputs(case)
    torch.set_num_threads(os.cpu_count())
    orc = po.Oracle(sd, cfg)
    P = cfg['patch_process_shape']
    H, W = case['image_raw_shape']
    h, w = H // 2, W // 2
    raw = [(0, 0), (h // 2, w // 2)]
    with torch.no_grad():
        lr = orc.resizer(img)
        d_o, f_o = orc.coarse(lr)
        g2l = po.g2l_all(sd, f_o, cfg['guided_fusion'])
        crops = torch.cat([orc.resizer(img[:, :, y:y + h, x:x + w]) for (y, x) in raw])
        fx, fy = 1 / W * P[1], 1 / H * P[0]
        boxes = torch.tensor([[x, y, x + w, y + h] for (y, x) in raw]).int() * torch.tensor([[fx, fy, fx, fy]])
        fd, ff = po.branch_forward(sd, 'fine_branch.', crops, cfg['fine_branch'])
        rois = [po.roi_crop_zoom(f, boxes, f.shape[-2] / P[0]) for f in f_o]
        droi = po.roi_crop_zoom(d_o, boxes, 1.0)
        ref = po.fusion_forward(sd, cfg, fd, crops, ff, boxes, droi, rois, g2l)
        with fp8_ref.fp8_unet():
            f8 = po.fusion_forward(sd, cfg, fd, crops, ff, boxes, droi, rois, g2l)
    assert torch.isfinite(f8).all()
    err = (f8 - ref).abs()
    rng = (ref.max() - ref.min()).item()
    print('FP8-emulated U-Net vs fp32 oracle, vits_case0 two tiles: max-abs %.3e (/80 %.3e, /range %.3e), '
          'mean-abs %.3e, depth range %.3f..%.3f' % (err.max().item(), err.max().item() / 80, err.max().item() / rng,
                                                     err.mean().item(), ref.min().item(), ref.max().item()))
