"""vit_precision = 'fp8_static' on the GPU: the E4M3 ping-pong GEMM (pf_gemm_pp_e4m3_kernel) bit for bit on integer
probes at every ViT linear shape and output kind, an fp64 sweep, pf_layernorm_e4m3 against its torch restatement, each
E4M3 linear of a vitl branch on exactly the input it read, model parity against the FP8 emulation, the invariances,
calibration, launch counts, and no change to the bf16 / FP8 U-Net models."""
import json
import os
import random
import zlib

import pytest
import torch
import torch.nn.functional as F

import fp8_static_ref as sref
import fp8_vit_ref as vref
from test_gpu_fp8_static import _infer, _same, _units, _units8

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
MAX_DEPTH = 80.0
BOUND_UNITS = 32.0      # the FP8 accumulator bound (DESIGN.md section 3)
RANGE_BAR = 2e-2
DIMS = {'vits': 384, 'vitb': 768, 'vitl': 1024}
POISON_BF16, POISON_F32, POISON_U8 = 3.0, -5.0, 0x7F


def _gen(*key):
    return torch.Generator(device='cuda').manual_seed(zlib.crc32(repr(key).encode()))


def _int_operand(shape, g, dev):
    v = torch.randint(-2, 3, shape, generator=g, device=dev).float()
    return v * (torch.rand(shape, generator=g, device=dev) < 0.25)


# ---------------------------------------------------------------------------------------------------- exact probes
# (kind, K, N) of each ViT linear: qkv (Q|K bf16 + V^T), fc1 (the e4m3 operand of fc2; bf16 too), fc2 (gamma reduce-add)
def _linears(D):
    return [('qkv', D, 3 * D), ('fc1', D, 4 * D), ('fc2', 4 * D, D)]


ROWS = [1037, 4 * 1037, 9 * 1037, 100, 200, 300]     # M = 1037 B and ragged M below / between 128-row tiles
PROBES = [(enc, lin, M) for enc in DIMS for lin in ('qkv', 'fc1', 'fc2') for M in ROWS
          if enc == 'vitl' or M in (1037, 200)]


@pytest.mark.parametrize('probe', PROBES, ids=['%s-%s-%d' % p for p in PROBES])
def test_linear_e4m3_exact(cuda, probe):
    """Integer operands at amax 7 (r = 64, scale 2^-6; every weight row holds a -7, so its scale is 2^-6 too): every
    product and sum is exact in the FP8 accumulator, so each output equals the fp64 GEMM rounded once (bf16), added once
    (fp32 gamma update), or quantized at the next ratio (e4m3, next amax 28).  Rows past M stay poisoned."""
    from patchfusion_b200 import ops
    enc, lin, M = probe
    D = DIMS[enc]
    _, K, N = {l: (l, k, n) for l, k, n in _linears(D)}[lin]
    g = _gen('lin8', probe)
    x = _int_operand((M, K), g, cuda)
    x[0, 0] = 7.0
    w = _int_operand((N, K), g, cuda)
    w[:, 0] = -7.0
    b = torch.randint(-4, 5, (N,), generator=g, device=cuda).float()
    pw = ops.pack_weight_e4m3(w, b)
    pad = 131                                          # rows past M, poisoned
    q = sref.quantize(x, 7.0).view(torch.uint8)
    ref = F.linear(x.double(), w.double(), b.double())
    kinds = {'qkv': ('bf16', 'vt'), 'fc1': ('bf16', 'e4m3'), 'fc2': ('f32',)}[lin]
    for kind in kinds:
        if kind in ('bf16', 'vt'):
            out = torch.full((M + pad, N if kind == 'bf16' else 2 * D), POISON_BF16, dtype=torch.bfloat16, device=cuda)
            if kind == 'vt':
                seq = 1037 if M % 1037 == 0 else M
                Bv = (M + seq - 1) // seq
                seq_pad = (seq + 7) // 8 * 8
                vt = torch.full((Bv * D, seq_pad), POISON_BF16, dtype=torch.bfloat16, device=cuda)
                ops.linear_e4m3(pw, q, 7.0, out, vt=(vt, 2 * D, seq))
                got, want = out[:M].float(), ref[:, :2 * D].to(torch.bfloat16).float()
                v = ref[:, 2 * D:].to(torch.bfloat16).float()          # [M, D] -> [(b, dd), tok]
                tok = torch.arange(M, device=cuda)
                vwant = torch.full_like(vt, POISON_BF16, dtype=torch.float32)
                vwant.view(Bv, D, seq_pad)[tok // seq, :, tok % seq] = v
                vbad = (vt.float() != vwant).nonzero()
                assert vbad.numel() == 0, 'V^T: %d mismatches, first at %s' % (vbad.shape[0], vbad[0].tolist())
            else:
                ops.linear_e4m3(pw, q, 7.0, out)
                got, want = out[:M].float(), ref.to(torch.bfloat16).float()
            assert (out[M:] == POISON_BF16).all(), 'rows past M were written'
        elif kind == 'f32':
            x0 = torch.randint(-8, 9, (M + pad, N), generator=g, device=cuda).float()
            x0[M:] = POISON_F32
            out = x0.clone()
            gamma = torch.ones(N, device=cuda)
            ops.linear_e4m3(pw, q, 7.0, out, gamma=gamma)
            got, want = out[:M], (x0[:M].double() + ref).float()
            assert (out[M:] == POISON_F32).all(), 'rows past M were written'
        else:
            out = torch.full((M + pad, N + 16), POISON_U8, dtype=torch.uint8, device=cuda)
            ops.linear_e4m3(pw, q, 7.0, out[:, :N], out_amax=28.0)
            got = out[:M, :N].view(torch.float8_e4m3fn).float()
            want = sref.quantize(ref.float(), 28.0).float()
            assert (out[M:] == POISON_U8).all() and (out[:, N:] == POISON_U8).all(), 'bytes past the output were written'
        bad = (got != want).nonzero()
        assert bad.numel() == 0, '%s %s: %d mismatches, first at %s (got %s want %s)' % (
            probe, kind, bad.shape[0], bad[0].tolist(), got[tuple(bad[0])].item(), want[tuple(bad[0])].item())
        print('e4m3 linear exact %s %s: ok' % (probe, kind))


def test_linear_e4m3_refusals(cuda):
    from patchfusion_b200 import lib, ops
    g = _gen('refuse')
    w = torch.randn(256, 192, generator=g, device=cuda)
    pw = ops.pack_weight_e4m3(w, None)
    q = torch.zeros(300, 192, dtype=torch.uint8, device=cuda)
    with pytest.raises(lib.PFError, match='e4m3 linear'):      # K = 192: not a multiple of 128
        ops.linear_e4m3(pw, q, 1.0, torch.zeros(300, 256, dtype=torch.bfloat16, device=cuda))


# ---------------------------------------------------------------------------------------------------- fp64 sweep
SWEEP = [(enc, lin, M) for enc in ('vits', 'vitb', 'vitl') for lin in ('qkv', 'fc1', 'fc2') for M in (9 * 1037, 333)]


@pytest.mark.parametrize('case', SWEEP, ids=['%s-%s-%d' % c for c in SWEEP])
def test_linear_e4m3_fp64_sweep(cuda, case):
    """random operands against the fp64 GEMM of the dequantized operands: within the accumulator bound; an e4m3 output
    within that bound past its rounding (half an e4m3 step), and within one e4m3 step of its quantized reference
    wherever the bound is below half a step (near zero the bound's 2^-14-of-max term spans many subnormal steps)"""
    from patchfusion_b200 import ops
    enc, lin, M = case
    D = DIMS[enc]
    _, K, N = {l: (l, k, n) for l, k, n in _linears(D)}[lin]
    g = _gen('sweep8', case)
    x = torch.randn(M, K, generator=g, device=cuda) * 1.5
    amax = x.abs().max().item() * 0.8                      # some inputs saturate
    w = torch.randn(N, K, generator=g, device=cuda) * K ** -0.5
    b = torch.randn(N, generator=g, device=cuda) * 0.1
    pw = ops.pack_weight_e4m3(w, b)
    q = sref.quantize(x, amax).view(torch.uint8)
    ref = vref.linear_e4m3_f64(q, amax, w, b)
    if lin == 'fc2':
        out = torch.zeros(M, N, device=cuda)
        gamma = torch.rand(N, generator=g, device=cuda) + 0.5
        ops.linear_e4m3(pw, q, amax, out, gamma=gamma)
        u = _units(out / gamma, ref)
    else:
        out = torch.empty(M, N, dtype=torch.bfloat16, device=cuda)
        ops.linear_e4m3(pw, q, amax, out, act=ops.ACT_GELU if lin == 'fc1' else ops.ACT_NONE)
        want = F.gelu(ref) if lin == 'fc1' else ref
        u = _units(out.float(), want)
    print('%s: %.2f units' % (case, u))
    assert u <= BOUND_UNITS, u
    if lin == 'fc1':
        o8 = torch.empty(M, N, dtype=torch.uint8, device=cuda)
        out_amax = 2.0
        ops.linear_e4m3(pw, q, amax, o8, act=ops.ACT_GELU, out_amax=out_amax)
        gelu = F.gelu(ref)
        u8 = _units8(sref.dequantize(o8.view(torch.float8_e4m3fn), out_amax).double(), gelu.clamp(-out_amax, out_amax))
        got = o8.view(torch.float8_e4m3fn).double()
        wq = sref.quantize(gelu.float(), out_amax).double()
        step = torch.pow(2.0, torch.floor(torch.log2(wq.abs().clamp_min(2.0 ** -6))) - 3)
        # the accumulator bound in e4m3 units of this output: 32 x (1 bf16 ulp + 2^-14 of the largest value) x r
        bound = BOUND_UNITS * (torch.pow(2.0, torch.floor(torch.log2(gelu.abs().clamp_min(1e-30))) - 7) +
                               gelu.abs().max().item() * 2.0 ** -14) * (448.0 / out_amax)
        far = (got - wq).abs() > step
        print('e4m3 output: %.2f units past the rounding; %d of %d more than one step from the quantized reference'
              % (u8, far.sum().item(), far.numel()))
        assert u8 <= BOUND_UNITS, u8
        assert not (far & (bound < 0.5 * step)).any(), 'more than one step off where the bound is below half a step'


# ---------------------------------------------------------------------------------------------------- LayerNorm
@pytest.mark.parametrize('C', [384, 768, 1024])
def test_layernorm_e4m3(cuda, C):
    from patchfusion_b200 import ops
    g = _gen('ln8', C)
    rows = 9 * 1037 + 5
    x = torch.randn(rows, C, generator=g, device=cuda) * 3 + torch.randn(rows, 1, generator=g, device=cuda)
    w = torch.randn(C, generator=g, device=cuda)
    b = torch.randn(C, generator=g, device=cuda) * 0.1
    amax = 4.0
    out = torch.full((rows, C + 16), POISON_U8, dtype=torch.uint8, device=cuda)
    ops.layernorm_e4m3(x, w, b, 1e-6, amax, out)
    got = out[:, :C]
    want = vref.layernorm_e4m3(x, w, b, 1e-6, amax)
    diff = (got != want)
    gf, wf = got.view(torch.float8_e4m3fn).float(), want.view(torch.float8_e4m3fn).float()
    print('C %d: %d of %d entries differ from the torch restatement' % (C, diff.sum().item(), diff.numel()))
    assert not torch.isnan(gf).any()
    # a difference is a value on an e4m3 rounding boundary: the neighbouring code
    step = torch.pow(2.0, torch.floor(torch.log2(wf.abs().clamp_min(2.0 ** -6))) - 3)
    assert ((gf - wf).abs() <= step)[diff].all()
    assert diff.float().mean().item() < 1e-3
    assert (out[:, C:] == POISON_U8).all()
    # the bf16 LayerNorm's affine value is the same fp32 number: quantizing its bf16 rounding differs only by that rounding
    hb = torch.empty(rows, C, dtype=torch.bfloat16, device=cuda)
    ops.layernorm(x, w, b, 1e-6, hb)
    assert (hb.float() - vref.layernorm_f32(x, w, b, 1e-6)).abs().max().item() <= \
        (vref.layernorm_f32(x, w, b, 1e-6).abs().max().item() * 2 ** -8)


# ---------------------------------------------------------------------------------------------------- vits model
@pytest.fixture(scope='module')
def vits(cuda):
    from oracle.make_golden import case_inputs
    from patchfusion_b200.model import PatchFusion
    case = json.load(open(os.path.join(GOLD, 'vits_case0.json')))
    cfg, sd, img0 = case_inputs(case)
    shape = tuple(case['image_raw_shape'])
    imgs = torch.cat([img0] + [torch.rand(1, 3, *shape, generator=torch.Generator().manual_seed(s))
                               for s in (101, 202)]).to(cuda)

    def make(**kw):
        m = PatchFusion(dict(cfg, **kw))
        m.load_state_dict(sd, strict=True)
        return m.to(cuda).eval()
    cal = torch.rand(2, 3, *shape, generator=torch.Generator().manual_seed(7)).to(cuda)
    v8 = make(vit_precision='fp8_static')
    random.seed(1)
    vtable = v8.calibrate_fp8(v8.make_lr(cal), cal, cai_mode='r4', process_num=4)
    both = make(vit_precision='fp8_static', fusion_precision='fp8_static')
    random.seed(1)
    both.calibrate_fp8(both.make_lr(cal), cal, cai_mode='r4', process_num=4)
    lr = v8.make_lr(imgs)
    return dict(case=case, cfg=cfg, sd=sd, make=make, v8=v8, both=both, imgs=imgs, lr=lr, cal=cal, vtable=vtable)


def test_forward_without_table_refuses(cuda, vits):
    m = vits['make'](vit_precision='fp8_static')
    with pytest.raises(RuntimeError, match='calibrate_fp8'):
        m(mode='infer', image_lr=vits['lr'][:1], image_hr=vits['imgs'][:1], cai_mode='m1', process_num=2)


def test_calibration(cuda, vits):
    """deterministic, all 6 depth names, merged by max; both tables filled for a model with both precisions; a changed
    table re-points the stage (graphs recaptured) and equals a freshly built model with it"""
    from patchfusion_b200.params import FP8_LAYERS, vit_fp8_layers
    s = vits
    names = vit_fp8_layers(s['cfg'])
    assert len(names) == 72 and set(s['vtable']) == set(names) and all(v > 0 for v in s['vtable'].values())
    assert set(s['both'].config['vit_fp8_amax']) == set(names) and set(s['both'].config['fusion_fp8_amax']) == set(FP8_LAYERS)
    m = s['make'](vit_precision='fp8_static')
    a = m.calibrate_fp8(s['lr'][:1], s['imgs'][:1], cai_mode='m1', process_num=2)
    b = m.calibrate_fp8(s['lr'][:1], s['imgs'][:1], cai_mode='m1', process_num=2, reset=True)
    assert a == b and set(a) == set(names)
    m.calibrate_fp8(s['lr'][1:2], s['imgs'][1:2], cai_mode='m1', process_num=2)
    merged = dict(m.config['vit_fp8_amax'])
    two = m.calibrate_fp8(s['lr'][:2], s['imgs'][:2], cai_mode='m1', process_num=2, reset=True)
    assert merged == two
    # graphs captured with one table are dropped when the table changes; the result is a fresh model's with that table
    lr, img = s['lr'][:1], s['imgs'][:1]
    y0 = _infer(m, lr, img, 4, cai_mode='m2', process_num=4)
    _same('graph replay', _infer(m, lr, img, 4, cai_mode='m2', process_num=4), y0)
    m.config['vit_fp8_amax'] = dict(s['vtable'])
    y1 = _infer(m, lr, img, 4, cai_mode='m2', process_num=4)
    fresh = s['make'](vit_precision='fp8_static', vit_fp8_amax=dict(s['vtable']))
    _same('changed table vs fresh model', y1, _infer(fresh, lr, img, 4, cai_mode='m2', process_num=4))
    assert not torch.equal(y0, y1)


def test_model_vs_fp8_emulation(cuda, vits):
    from oracle import pf_oracle as po
    s = vits
    model, img, lr = s['v8'], s['imgs'][:1], s['lr'][:1]
    pn = s['case']['process_num']
    orc = po.Oracle({k: v.to(cuda) for k, v in s['sd'].items()}, s['cfg'])
    bf = s['make']()
    for mode in ('m1', 'm2', 'r4'):
        got = _infer(model, lr, img, 0, cai_mode=mode, process_num=pn)
        with torch.no_grad(), vref.fp8_static_vit(s['vtable']):
            random.seed(0)
            want = orc.infer(lr, img, cai_mode=mode, process_num=pn).to(got.device).view(got.shape)
        d16 = (got - _infer(bf, lr, img, 0, cai_mode=mode, process_num=pn)).abs()
        err, rng = (got - want).abs().max().item(), (want.max() - want.min()).item()
        print('%s: FP8 ViT vs FP8 emulation max-abs %.3e (/80 %.3e, /range %.3e); vs bf16 max %.3e mean %.3e'
              % (mode, err, err / MAX_DEPTH, err / rng, d16.max().item(), d16.mean().item()))
        assert torch.isfinite(got).all()
        assert err / MAX_DEPTH < 1e-3, mode


@pytest.mark.parametrize('which', ['v8', 'both'])
def test_invariances(cuda, vits, which):
    s = vits
    model, lr, imgs = s[which], s['lr'], s['imgs']
    _same('%s m2 process_num 9 vs 4' % which, _infer(model, lr[:1], imgs[:1], 3, cai_mode='m2', process_num=9),
          _infer(model, lr[:1], imgs[:1], 3, cai_mode='m2', process_num=4))
    for mode in ('m2', 'r4'):
        random.seed(5)
        want = torch.cat([model(mode='infer', image_lr=lr[b:b + 1], image_hr=imgs[b:b + 1], cai_mode=mode,
                                process_num=2)[0].clone() for b in range(imgs.shape[0])])
        _same('%s %s B=3 vs 3 x B=1' % (which, mode), _infer(model, lr, imgs, 5, cai_mode=mode, process_num=2), want)
        _same('%s %s emulated world 8' % (which, mode),
              _infer(model, lr, imgs, 5, cai_mode=mode, process_num=2, shard=('emulate', 8)), want)
    shapes = [((1080, 1920), (2, 2)), ((720, 1280), (2, 4)), ((540, 960), (1, 1))]
    mi = [torch.rand(1, 3, *hw, generator=torch.Generator().manual_seed(10 + i)).to(cuda)
          for i, (hw, _) in enumerate(shapes)]
    cfgs = [{'image_raw_shape': list(hw), 'patch_split_num': list(p)} for hw, p in shapes]
    mlr = model.make_lr(mi)
    modes = ['m2', 'r4', 'm1']
    random.seed(7)
    want = [model(mode='infer', image_lr=mlr[b:b + 1], image_hr=mi[b], tile_cfg=cfgs[b], cai_mode=modes[b],
                  process_num=9)[0].clone() for b in range(3)]
    random.seed(7)
    got, _ = model(mode='infer', image_lr=mlr, image_hr=mi, tile_cfg=cfgs, cai_mode=modes, process_num=9)
    for b in range(3):
        _same('%s mixed geometry image %d' % (which, b), got[b], want[b])


def _profiled_names(model, lr, img):
    from patchfusion_b200 import lib
    prof = lib.Profiler()
    lib.PROFILER = prof
    try:
        prof.start()
        _infer(model, lr, img, 1, cai_mode='m1', process_num=2)
        recs = prof.stop()
    finally:
        lib.PROFILER = None
    return [r[0] for r in recs]


def test_launches(cuda, vits):
    """per branch call: 3 depth e4m3 GEMMs, 2 depth e4m3 LayerNorms, no quantize launch for the ViT"""
    s = vits
    depth = 12
    for which, unet_q in (('v8', 0), ('both', 17)):
        names = _profiled_names(s[which], s['lr'][:1], s['imgs'][:1])
        calls = names.count('assemble_tokens_kernel')
        fus = names.count('pack_unet_input_kernel')
        n8, nl = names.count('pf_gemm_pp_e4m3_kernel'), names.count('layernorm_e4m3_kernel')
        print('%s m1: %d branch calls, %d e4m3 GEMMs, %d e4m3 LayerNorms' % (which, calls, n8, nl))
        assert calls > 0 and n8 == 3 * depth * calls and nl == 2 * depth * calls
        assert names.count('quant_static_kernel') == unet_q * fus
        assert names.count('quant_amax_kernel') == 0 and names.count('quant_write_kernel') == 0
        ref = s['make'](fusion_precision='fp8_static' if which == 'both' else 'bf16',
                        fusion_fp8_amax=s['both'].config['fusion_fp8_amax'] if which == 'both' else None)
        _infer(ref, s['lr'][:1], s['imgs'][:1], 1, cai_mode='m1', process_num=2)       # packs its weights first
        bf_names = _profiled_names(ref, s['lr'][:1], s['imgs'][:1])
        # each e4m3 GEMM replaces a bf16 one, each e4m3 LayerNorm a bf16 one: the same launch count
        assert len(names) == len(bf_names)


def _count(model, lr, img):
    from patchfusion_b200 import lib
    torch.cuda.synchronize()
    n0 = lib.launch_count()
    y = _infer(model, lr, img, 9, cai_mode='m2', process_num=4)
    torch.cuda.synchronize()
    return y, lib.launch_count() - n0


def test_default_paths_unaffected(cuda, vits):
    """bf16 and both FP8 U-Net models: no new kernel, the same launch counts, workspace sizes and output bits next to
    an FP8 ViT model"""
    s = vits
    lr, img = s['lr'][:1], s['imgs'][:1]
    for prec in ('bf16', 'fp8', 'fp8_static'):
        kw = dict(fusion_precision=prec)
        if prec == 'fp8_static':
            kw['fusion_fp8_amax'] = dict(s['both'].config['fusion_fp8_amax'])
        m = s['make'](**kw)
        _infer(m, lr, img, 9, cai_mode='m2', process_num=4)
        before, n = _count(m, lr, img)
        names = _profiled_names(m, lr, img)
        assert 'pf_gemm_pp_e4m3_kernel' not in names and 'layernorm_e4m3_kernel' not in names
        y8 = _infer(s['v8'], lr, img, 9, cai_mode='m2', process_num=4)
        assert not torch.equal(y8, before)
        after, n2 = _count(m, lr, img)
        _same('%s model before / after an FP8 ViT model' % prec, after, before)
        assert n2 == n
    eb, e8 = s['make']().engine(), s['v8'].engine()
    for which in ('coarse', 'fine'):
        # the FP8 branch adds its two e4m3 operand buffers; the bf16 branch is the bf16 model's
        assert e8.branch_bytes(which, 4) > eb.branch_bytes(which, 4)
        from patchfusion_b200 import stage
        assert stage.branch_workspace_bytes(e8.c_branch_bf16[which], 4) == eb.branch_bytes(which, 4)


# ---------------------------------------------------------------------------------------------------- vitl branch
@pytest.fixture(scope='module')
def vitl_fine(cuda):
    from oracle import pf_oracle as po
    from oracle.make_golden import case_inputs
    from patchfusion_b200.model import PatchFusion
    case = json.load(open(os.path.join(GOLD, 'vitl_tile0.json')))
    cfg, sd, img = case_inputs(case)
    model = PatchFusion(dict(cfg, vit_precision='fp8_static'))
    model.load_state_dict(sd, strict=True)
    model = model.to(cuda).eval()
    eng = model.engine()
    sdc = {k: v.to(cuda) for k, v in sd.items()}
    img = img.to(cuda)
    H, W = case['image_raw_shape']
    th, tw = case.get('tile', (H // 2, W // 2))
    orc = po.Oracle(sdc, cfg)
    with torch.no_grad():
        crops = torch.cat([orc.resizer(img[:, :, y:y + th, x:x + tw]) for (y, x) in [(0, 0), (H - th, W - tw)]])
        crops = crops.contiguous()
        eng.calib = {}                                   # calibrate the fine encoder on these two tiles
        eng.branch('fine', crops)
        fine = {k: v.item() for k, v in eng.calib.items()}
        eng.calib = None
        eng.calib = {}
        eng.branch('coarse', crops[:1].contiguous())
        coarse = {k: v.item() for k, v in eng.calib.items()}
        eng.calib = None
        table = dict(fine, **coarse)
        eng.set_vit_fp8_amax(table)
        taps = {}
        got, _ = eng.branch('fine', crops, taps)
        got = got.clone()
        with vref.fp8_static_vit(table):
            want, _ = po.branch_forward(sdc, 'fine_branch.', crops, cfg['fine_branch'])
        torch.cuda.synchronize()
    return dict(sd=sdc, taps=taps, table=table, got=got, want=want[:, 0], cfg=cfg)


def test_vitl_each_linear_on_its_own_input(cuda, vitl_fine):
    s = vitl_fine
    taps, table = s['taps'], s['table']
    pre = 'fine_branch.core.core.pretrained.blocks.%d.'
    D = 1024
    worst = {}
    for i in range(24):
        w = lambda n: s['sd'][pre % i + n]
        am = {k: table['fine.%d.%s' % (i, k)] for k in ('qkv', 'fc1', 'fc2')}
        ref = vref.linear_e4m3_f64(taps['e4m3v.%d.qkv.in' % i], am['qkv'], w('attn.qkv.weight'), w('attn.qkv.bias'))
        u_qk = _units(taps['e4m3v.%d.qkv.out' % i].float(), ref[:, :2 * D])
        rows = ref.shape[0]
        seq = rows // 2
        vt = taps['e4m3v.%d.qkv.vt' % i].float().view(2, D, -1)[:, :, :seq].permute(0, 2, 1).reshape(rows, D)
        u_v = _units(vt, ref[:, 2 * D:])
        ref1 = F.gelu(vref.linear_e4m3_f64(taps['e4m3v.%d.fc1.in' % i], am['fc1'], w('mlp.fc1.weight'), w('mlp.fc1.bias')))
        got1 = sref.dequantize(taps['e4m3v.%d.fc1.out' % i].view(torch.float8_e4m3fn), am['fc2']).double()
        u_1 = _units8(got1, ref1.clamp(-am['fc2'], am['fc2']))
        ref2 = vref.linear_e4m3_f64(taps['e4m3v.%d.fc2.in' % i], am['fc2'], w('mlp.fc2.weight'), w('mlp.fc2.bias'))
        delta = (taps['e4m3v.%d.fc2.out' % i].double() - taps['e4m3v.%d.fc2.x' % i].double()) / w('ls2.gamma').double()
        u_2 = _units(delta, ref2)
        worst[i] = (u_qk, u_v, u_1, u_2)
        assert max(u_qk, u_v, u_2) <= BOUND_UNITS and u_1 <= BOUND_UNITS, (i, worst[i])
    print('vitl 4K fine branch, worst units per linear (qk, v, fc1, fc2): %s' %
          str(tuple(max(v[j] for v in worst.values()) for j in range(4))))


def test_vitl_branch_vs_fp8_emulation(cuda, vitl_fine):
    s = vitl_fine
    got, want = s['got'], s['want']
    err, rng = (got - want).abs().max().item(), (want.max() - want.min()).item()
    print('vitl fine branch: FP8 ViT vs FP8 emulation max-abs %.3e (/80 %.3e, /range %.3e)'
          % (err, err / MAX_DEPTH, err / rng))
    assert torch.isfinite(got).all()
    assert err / MAX_DEPTH < 1e-3
    if err / rng >= RANGE_BAR:
        pytest.xfail('%.1f %% of the output range, above the 2 %% bar (synthetic weights)' % (100 * err / rng))
