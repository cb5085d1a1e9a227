"""dpt_precision = 'fp8_static' on the GPU: pf_conv3_halo_e4m3_res_kernel bit for bit on integer probes (residuals, the
e4m3 ReLU copy, poisoned edges), an fp64 sweep at the DPT conv shapes, each covered conv of a vitl fine branch on exactly
its own inputs, model parity against the FP8 emulation, the invariances, calibration, launch counts, and no change to
the bf16 model."""
import json
import os
import random
import zlib

import pytest
import torch
import torch.nn.functional as F

import fp8_dpt_ref as dref
import fp8_static_ref as sref
from test_gpu_fp8_static import _infer, _same, _units

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
MAX_DEPTH = 80.0
BOUND_UNITS = 32.0      # the FP8 accumulator bound (DESIGN.md section 3)
RANGE_BAR = 2e-2
POISON_BF16, POISON_U8 = 3.0, 0x7F


def _gen(*key):
    return torch.Generator(device='cuda').manual_seed(zlib.crc32(repr(key).encode()))


def _int_operand(shape, g, dev, p=0.25):
    v = torch.randint(-2, 3, shape, generator=g, device=dev).float()
    return v * (torch.rand(shape, generator=g, device=dev) < p)


def _pad(n, m):
    return (n + m - 1) // m * m


# ---------------------------------------------------------------------------------------------------- exact probes
# (C_in, N, T, H, W): N = C of vits / vitb / vitl (64 / 128 / 256: BN 64 / 128 / two 128 tiles), a narrow N with pad
# columns in the copy, partial 16 x 8 pixel tiles, and a micro-batch with weight-multicast clusters
PROBES = [(64, 64, 2, 19, 23), (128, 128, 3, 16, 8), (256, 256, 2, 17, 29), (256, 256, 9, 56, 74), (64, 40, 2, 9, 13)]
KINDS = [(False, False), (True, False), (False, True), (True, True)]       # (res2, copy); res1 always


@pytest.mark.parametrize('kind', KINDS, ids=['r1', 'r2', 'r1-copy', 'r2-copy'])
@pytest.mark.parametrize('probe', PROBES, ids=['%d-%d-%d-%dx%d' % p for p in PROBES])
def test_res_conv_exact(cuda, probe, kind):
    """Integer operands at amax 7 (r = 64, scale 2^-6) and integer residuals: the accumulator, the bias add and both
    residual adds are exact, so the bf16 output is the fp64 sum rounded once, and the copy is the static quantize of
    its ReLU at amax 28 (r = 16, past 28 saturates).  Columns past N of the bf16 output and bytes past the copy's padded
    width stay poisoned; the copy's pad columns are zero."""
    from patchfusion_b200 import ops
    C, N, T, H, W = probe
    res2_on, copy_on = kind
    g = _gen('res8', probe, kind)
    x = _int_operand((T, H, W, C), g, cuda)
    x[:, 0, 0, 0] = 7.0
    w = _int_operand((N, C, 3, 3), g, cuda)
    w[:, 0, 2, 2] = -7.0
    b = torch.randint(-4, 5, (N,), generator=g, device=cuda).float()
    pw = ops.pack_weight_e4m3(w, b)
    xb = torch.zeros((T, H, W, _pad(C, 8)), dtype=torch.bfloat16, device=cuda)
    xb[..., :C] = x
    q = ops.quantize_e4m3_static([xb], 7.0)
    ld = _pad(N, 8)
    r1 = (torch.randint(-40, 41, (T, H, W, ld), generator=g, device=cuda).float()).bfloat16()
    r2 = (torch.randint(-40, 41, (T, H, W, ld), generator=g, device=cuda).float()).bfloat16() if res2_on else None
    ref = F.conv2d(x.permute(0, 3, 1, 2).double(), w.double(), b.double(), padding=1).permute(0, 2, 3, 1)
    ref = ref + r1[..., :N].double() + (r2[..., :N].double() if res2_on else 0)
    out = torch.full((T, H, W, ld), POISON_BF16, dtype=torch.bfloat16, device=cuda)
    kc = _pad(N, 64)
    copy = torch.full((T, H, W, kc + 16), POISON_U8, dtype=torch.uint8, device=cuda) if copy_on else None
    d = ops.conv3_e4m3_static(pw, q, 7.0, out, act=0, res1=r1, res2=r2, copy=copy, copy_amax=28.0)
    want = ref.to(torch.bfloat16)
    bad = (out[..., :N] != want).nonzero()
    assert bad.numel() == 0, 'block_n %d: %d mismatches, first at %s (got %s want %s)' % (
        d.block_n, bad.shape[0], bad[0].tolist(), out[tuple(bad[0])].item(), want[tuple(bad[0])].item())
    if ld > N:
        assert (out[..., N:] == POISON_BF16).all(), 'columns past N were written'
    if copy_on:
        got = copy[..., :kc].view(torch.float8_e4m3fn).float()
        wq = torch.zeros_like(got)
        wq[..., :N] = sref.quantize(F.relu(out[..., :N].float()), 28.0).float()
        assert torch.equal(got, wq), 'e4m3 copy differs from the static quantize of relu(out)'
        assert (copy[..., kc:] == POISON_U8).all(), 'bytes past the padded width were written'
        assert (got.abs() == 448).any() or N < 64, 'no saturated value in the probe'
    print('res probe C %d N %d T %d %dx%d res2 %s copy %s: block_n %d ok' % (C, N, T, H, W, res2_on, copy_on, d.block_n))


def test_res_conv_refusals(cuda):
    from patchfusion_b200 import lib, ops
    pw = ops.pack_weight_e4m3(torch.randn(64, 64, 3, 3, device=cuda), None)
    q = ops.quantize_e4m3_static([torch.randn(1, 8, 8, 64, device=cuda).bfloat16()], 1.0)
    out = torch.zeros(1, 8, 8, 64, dtype=torch.bfloat16, device=cuda)
    r = torch.zeros_like(out)
    with pytest.raises(lib.PFError):            # an e4m3 main output with residuals
        ops.conv3_e4m3_static(pw, q, 1.0, torch.zeros(1, 8, 8, 64, dtype=torch.uint8, device=cuda), next_amax=1.0, res1=r)
    with pytest.raises(lib.PFError):            # a copy map narrower than 64 ceil(N / 64)
        ops.conv3_e4m3_static(pw, q, 1.0, out, res1=r, copy=torch.zeros(1, 8, 8, 48, dtype=torch.uint8, device=cuda),
                              copy_amax=1.0)
    with pytest.raises(lib.PFError):            # block_n 192 has no residual instantiation
        ops.conv3_e4m3_static(pw, q, 1.0, out, res1=r, block_n=192)


# ---------------------------------------------------------------------------------------------------- fp64 sweep
def _dpt_shapes(enc):
    """(name, C_in, N, H, W) of the 19 covered convs of a 392 x 518 branch"""
    from patchfusion_b200.params import branch_hparams
    from patchfusion_b200.configs import depth_anything_patchfusion
    cfg = depth_anything_patchfusion(enc, image_raw_shape=[2160, 3840], patch_split_num=[4, 4])
    hp = branch_hparams(cfg['fine_branch'])
    C, oc = hp['features'], hp['out_channels']
    gh, gw = 392 // 14, 518 // 14
    sizes = [(gh * 4, gw * 4), (gh * 2, gw * 2), (gh, gw), ((gh - 1) // 2 + 1, (gw - 1) // 2 + 1)]
    out = [('layer%d_rn' % (i + 1), oc[i], C) + sizes[i] for i in range(4)]
    for i in (1, 2, 3):
        out += [('refinenet%d.rcu' % i, C, C) + sizes[i - 1]]
    out += [('refinenet4.rcu', C, C) + sizes[3], ('output_conv1', C, C // 2, gh * 8, gw * 8)]
    return out


SWEEP = [(enc,) + s for enc in ('vits', 'vitl') for s in _dpt_shapes(enc)]


@pytest.mark.parametrize('case', SWEEP, ids=['%s-%s' % (c[0], c[1]) for c in SWEEP])
def test_res_conv_fp64_sweep(cuda, case):
    """random activations at micro-batch 9 through the conv each shape runs as (reassemble: copy, no residual; RCU
    conv2: two residuals and the copy; output_conv1: the q8 kernel), against an fp64 conv of the dequantized operands plus
    the residuals: within the accumulator bound"""
    from patchfusion_b200 import ops
    enc, name, C, N, H, W = case
    T = 9
    g = _gen('sweep8', case)
    x = (torch.randn(T, H, W, C, generator=g, device=cuda) * 2).bfloat16()
    w = torch.randn(N, C, 3, 3, generator=g, device=cuda) / (3 * C ** 0.5)
    b = torch.randn(N, generator=g, device=cuda) * 0.1
    amax = x.float().abs().max().item()
    pw = ops.pack_weight_e4m3(w, b)
    q = ops.quantize_e4m3_static([x.contiguous()], amax)
    out = torch.zeros(T, H, W, N, dtype=torch.bfloat16, device=cuda)
    ref = dref.conv_e4m3_f64(q, amax, w, b)
    r1 = r2 = copy = None
    if name.endswith('rcu'):
        r1 = torch.randn(T, H, W, N, generator=g, device=cuda).bfloat16()
        r2 = torch.randn(T, H, W, N, generator=g, device=cuda).bfloat16()
        ref = ref + r1.double() + r2.double()
    if name != 'output_conv1':
        copy = torch.zeros(T, H, W, _pad(N, 64), dtype=torch.uint8, device=cuda)
    ops.conv3_e4m3_static(pw, q, amax, out, act=0, res1=r1, res2=r2, copy=copy, copy_amax=3.0)
    u = _units(out.float(), ref)
    print('%s %s %dx%d C %d N %d: %.2f units' % (enc, name, H, W, C, N, u))
    assert u <= BOUND_UNITS
    if copy is not None:
        assert torch.equal(copy[..., :N], sref.quantize(F.relu(out.float()), 3.0).view(torch.uint8))


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
    d8 = make(dpt_precision='fp8_static')
    random.seed(1)
    dtable = d8.calibrate_fp8(d8.make_lr(cal), cal, cai_mode='r4', process_num=4)
    allm = make(dpt_precision='fp8_static', vit_precision='fp8_static', fusion_precision='fp8_static')
    random.seed(1)
    allm.calibrate_fp8(allm.make_lr(cal), cal, cai_mode='r4', process_num=4)
    lr = d8.make_lr(imgs)
    return dict(case=case, cfg=cfg, sd=sd, make=make, d8=d8, all=allm, imgs=imgs, lr=lr, cal=cal, dtable=dtable)


def test_forward_without_table_refuses(cuda, vits):
    m = vits['make'](dpt_precision='fp8_static')
    with pytest.raises(RuntimeError, match='calibrate_fp8'):
        m(mode='infer', image_lr=vits['lr'][:1], image_hr=vits['imgs'][:1], cai_mode='m1', process_num=2)


def test_calibration(cuda, vits):
    """all 38 names, deterministic, merged by max; all three tables for a model with all three keys; a changed table
    re-points the stage (graphs recaptured) and equals a freshly built model with it"""
    from patchfusion_b200.params import FP8_LAYERS, dpt_fp8_layers, vit_fp8_layers
    s = vits
    names = dpt_fp8_layers(s['cfg'])
    assert len(names) == 38 and set(s['dtable']) == set(names) and all(v > 0 for v in s['dtable'].values())
    c = s['all'].config
    assert set(c['dpt_fp8_amax']) == set(names) and set(c['fusion_fp8_amax']) == set(FP8_LAYERS)
    assert set(c['vit_fp8_amax']) == set(vit_fp8_layers(s['cfg']))
    m = s['make'](dpt_precision='fp8_static')
    a = m.calibrate_fp8(s['lr'][:1], s['imgs'][:1], cai_mode='m1', process_num=2)
    b = m.calibrate_fp8(s['lr'][:1], s['imgs'][:1], cai_mode='m1', process_num=2, reset=True)
    assert a == b and set(a) == set(names)
    m.calibrate_fp8(s['lr'][1:2], s['imgs'][1:2], cai_mode='m1', process_num=2)
    merged = dict(m.config['dpt_fp8_amax'])
    two = m.calibrate_fp8(s['lr'][:2], s['imgs'][:2], cai_mode='m1', process_num=2, reset=True)
    assert merged == two
    lr, img = s['lr'][:1], s['imgs'][:1]
    y0 = _infer(m, lr, img, 4, cai_mode='m2', process_num=4)
    _same('graph replay', _infer(m, lr, img, 4, cai_mode='m2', process_num=4), y0)
    m.config['dpt_fp8_amax'] = dict(s['dtable'])
    y1 = _infer(m, lr, img, 4, cai_mode='m2', process_num=4)
    fresh = s['make'](dpt_precision='fp8_static', dpt_fp8_amax=dict(s['dtable']))
    _same('changed table vs fresh model', y1, _infer(fresh, lr, img, 4, cai_mode='m2', process_num=4))
    assert not torch.equal(y0, y1)


def test_model_vs_fp8_emulation(cuda, vits):
    from oracle import pf_oracle as po
    s = vits
    model, img, lr = s['d8'], s['imgs'][:1], s['lr'][:1]
    pn = s['case']['process_num']
    orc = po.Oracle({k: v.to(cuda) for k, v in s['sd'].items()}, s['cfg'])
    bf = s['make']()
    worst = 0.0
    for mode in ('m1', 'm2', 'r4'):
        got = _infer(model, lr, img, 0, cai_mode=mode, process_num=pn)
        with torch.no_grad(), dref.fp8_static_dpt(s['dtable']):
            random.seed(0)
            want = orc.infer(lr, img, cai_mode=mode, process_num=pn).to(got.device).view(got.shape)
        d16 = (got - _infer(bf, lr, img, 0, cai_mode=mode, process_num=pn)).abs()
        err, rng = (got - want).abs().max().item(), (want.max() - want.min()).item()
        worst = max(worst, err / rng)
        print('%s: FP8 DPT vs FP8 emulation max-abs %.3e (/80 %.3e, /range %.3e); vs bf16 max %.3e mean %.3e'
              % (mode, err, err / MAX_DEPTH, err / rng, d16.max().item(), d16.mean().item()))
        assert torch.isfinite(got).all()
        assert err / MAX_DEPTH < 1e-3, mode
    if worst >= RANGE_BAR:
        pytest.xfail('%.1f %% of the output range, above the 2 %% bar (synthetic weights)' % (100 * worst))


@pytest.mark.parametrize('which', ['d8', 'all'])
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
    """per branch call: 19 E4M3 DPT convs (11 with residuals / a copy, 8 on the q8 kernel: the 7 RCU conv1s and
    output_conv1) and 5 static quantizes, exactly 5 launches more than bf16"""
    s = vits
    names = _profiled_names(s['d8'], s['lr'][:1], s['imgs'][:1])
    calls = names.count('assemble_tokens_kernel')
    nres, nq8 = names.count('pf_conv3_halo_e4m3_res_kernel'), names.count('pf_conv3_halo_e4m3_q8_kernel')
    nquant = names.count('quant_static_kernel')
    print('d8 m1: %d branch calls, %d res convs, %d q8 convs, %d static quantizes' % (calls, nres, nq8, nquant))
    assert calls > 0 and nres == 11 * calls and nq8 == 8 * calls and nquant == 5 * calls
    bf = s['make']()
    _infer(bf, s['lr'][:1], s['imgs'][:1], 1, cai_mode='m1', process_num=2)
    bf_names = _profiled_names(bf, s['lr'][:1], s['imgs'][:1])
    assert len(names) == len(bf_names) + 5 * calls


def _count(model, lr, img):
    from patchfusion_b200 import lib
    torch.cuda.synchronize()
    n0 = lib.launch_count()
    y = _infer(model, lr, img, 9, cai_mode='m2', process_num=4)
    torch.cuda.synchronize()
    return y, lib.launch_count() - n0


def test_default_paths_unaffected(cuda, vits):
    """a bf16 model next to an FP8 DPT model: no new kernel, the same launch count, workspace and output bits; the FP8
    model's bf16 branch structs (calibration) are the bf16 model's"""
    from patchfusion_b200 import stage
    s = vits
    lr, img = s['lr'][:1], s['imgs'][:1]
    for kw in ({}, {'dpt_precision': 'bf16'}):
        m = s['make'](**kw)
        _infer(m, lr, img, 9, cai_mode='m2', process_num=4)
        before, n = _count(m, lr, img)
        names = _profiled_names(m, lr, img)
        assert 'pf_conv3_halo_e4m3_res_kernel' not in names and 'quant_static_kernel' not in names
        y8 = _infer(s['d8'], lr, img, 9, cai_mode='m2', process_num=4)
        assert not torch.equal(y8, before)
        after, n2 = _count(m, lr, img)
        _same('bf16 model before / after an FP8 DPT model', after, before)
        assert n2 == n
    eb, e8 = s['make']().engine(), s['d8'].engine()
    for which in ('coarse', 'fine'):
        assert stage.branch_workspace_bytes(e8.c_branch_bf16[which], 4) == eb.branch_bytes(which, 4)


# ---------------------------------------------------------------------------------------------------- vitl branch
@pytest.fixture(scope='module')
def vitl_fine(cuda):
    from oracle import pf_oracle as po
    from oracle.make_golden import case_inputs
    from patchfusion_b200.model import PatchFusion
    case = json.load(open(os.path.join(GOLD, 'vitl_tile0.json')))
    cfg, sd, img = case_inputs(case)
    model = PatchFusion(dict(cfg, dpt_precision='fp8_static'))
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
        table = {}
        for which, x in (('fine', crops), ('coarse', crops[:1].contiguous())):
            eng.calib = {}
            eng.branch(which, x)
            table.update({k: v.item() for k, v in eng.calib.items()})
            eng.calib = None
        eng.set_dpt_fp8_amax(table)
        taps = {}
        got, _ = eng.branch('fine', crops, taps)
        got = got.clone()
        with dref.fp8_static_dpt(table):
            want, _ = po.branch_forward(sdc, 'fine_branch.', crops, cfg['fine_branch'])
        torch.cuda.synchronize()
    return dict(sd=sdc, taps=taps, table=table, got=got, want=want[:, 0], cfg=cfg, P=eng.P)


def test_vitl_exact_layer_set(cuda, vitl_fine):
    from patchfusion_b200.params import DPT_FP8_CONVS
    convs = {k[len('e4m3d.'):-len('.in')] for k in vitl_fine['taps'] if k.startswith('e4m3d.') and k.endswith('.in')}
    assert convs == set(DPT_FP8_CONVS)
    assert set(vitl_fine['table']) == {'%s.%s' % (b, n) for b in ('coarse', 'fine') for n in DPT_FP8_CONVS}


def test_vitl_each_conv_on_its_own_input(cuda, vitl_fine):
    """each covered conv against an fp64 conv of its tapped e4m3 input plus its tapped residuals: within the
    accumulator bound; each e4m3 ReLU copy equals the static quantize of that conv's bf16 output's ReLU"""
    from patchfusion_b200.params import DPT_FP8_CONVS
    s = vitl_fine
    taps, table = s['taps'], s['table']
    pre = 'fine_branch.core.core.depth_head.scratch.'
    worst = {}
    for n in DPT_FP8_CONVS:
        w = s['sd'][pre + n + '.weight']
        b = s['sd'].get(pre + n + '.bias')
        q = taps['e4m3d.%s.in' % n]
        rows = q.shape[0]
        B = 2
        hw = rows // B
        # recover the map's H x W from the branch geometry: the conv's rows are B x H x W
        H, W = _hw_of(n, hw, s['P'])
        ref = dref.conv_e4m3_f64(q.view(B, H, W, -1), table['fine.' + n], w, b).reshape(rows, -1)
        for r in ('res1', 'res2'):
            if 'e4m3d.%s.%s' % (n, r) in taps:
                ref = ref + taps['e4m3d.%s.%s' % (n, r)].double()
        out = taps['e4m3d.%s.out' % n]
        if n.endswith('conv1') and 'resConfUnit' in n:
            # conv1 writes conv2's e4m3 operand from relu(v): compare the dequantized bytes with half an e4m3 step
            nxt = table['fine.' + n[:-1] + '2']
            got = sref.dequantize(out[:, :w.shape[0]].view(torch.float8_e4m3fn), nxt).double()
            want = F.relu(ref).clamp(max=nxt)
            from test_gpu_fp8_static import _units8
            u = _units8(got, want)
        else:
            u = _units(out.float(), ref)
        worst[n] = u
        if 'e4m3d.%s.copy' % n in taps:
            reader = 'refinenet4.resConfUnit2.conv1' if n == 'layer4_rn' else (
                'refinenet%s.resConfUnit1.conv1' % n[5] if n.endswith('_rn') else n.replace('Unit1.conv2', 'Unit2.conv1'))
            cp = taps['e4m3d.%s.copy' % n][:, :w.shape[0]]
            assert torch.equal(cp, sref.quantize(F.relu(out.float()), table['fine.' + reader]).view(torch.uint8)), n
        assert u <= BOUND_UNITS, (n, u)
    print('vitl 4K fine branch, units per DPT conv: %s' % ', '.join('%s %.2f' % kv for kv in worst.items()))


def _hw_of(name, hw, P):
    gh, gw = P[0] // 14, P[1] // 14
    sizes = {1: (gh * 4, gw * 4), 2: (gh * 2, gw * 2), 3: (gh, gw), 4: ((gh - 1) // 2 + 1, (gw - 1) // 2 + 1)}
    if name == 'output_conv1':
        h, w = gh * 8, gw * 8
    elif name.endswith('_rn'):
        h, w = sizes[int(name[5])]
    else:
        h, w = sizes[int(name[len('refinenet')])]
    assert h * w == hw, (name, h, w, hw)
    return h, w


def test_vitl_branch_vs_fp8_emulation(cuda, vitl_fine):
    s = vitl_fine
    got, want = s['got'], s['want']
    err, rng = (got - want).abs().max().item(), (want.max() - want.min()).item()
    print('vitl fine branch: FP8 DPT vs FP8 emulation max-abs %.3e (/80 %.3e, /range %.3e)'
          % (err, err / MAX_DEPTH, err / rng))
    assert torch.isfinite(got).all()
    assert err / MAX_DEPTH < 1e-3
    if err / rng >= RANGE_BAR:
        pytest.xfail('%.1f %% of the output range, above the 2 %% bar (synthetic weights)' % (100 * err / rng))
