"""fusion_precision = 'fp8_static' on the GPU: pf_quantize_e4m3_static and the static-scale E4M3 conv (bf16 and e4m3
outputs) bit for bit against tests/fp8_static_ref.py, calibration against the 'fp8' path's own per-tile amaxes, each
static conv of a vitl 4K fusion stage on exactly the input it read, model parity against the static emulation, the
project's invariances, launch counts, and no state leaking into 'bf16' / 'fp8' models."""
import json
import os
import random
import zlib

import pytest
import torch
import torch.nn.functional as F

import fp8_ref
import fp8_static_ref as sref

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
MAX_DEPTH = 80.0
BOUND_UNITS = 32.0      # the FP8 accumulator bound of tests/test_gpu_fp8.py
RANGE_BAR = 2e-2
UNET_ORDER = (['inc.0', 'inc.1'] + ['down%d.%d' % (i, j) for i in range(5) for j in (0, 1)] + ['cv0.0', 'cv0.1'] +
              [n for i in range(1, 6) for n in ('up%d.0' % i, 'up%d.1' % i, 'cv%d.0' % i, 'cv%d.1' % i)])


def _gen(*key):
    return torch.Generator(device='cuda').manual_seed(zlib.crc32(repr(key).encode()))


def _same(tag, a, b):
    assert a.shape == b.shape, (tag, a.shape, b.shape)
    d = (a.float() - b.float()).abs().max().item()
    print('%s: max diff %.3e' % (tag, d))
    assert torch.isfinite(a.float()).all() and torch.isfinite(b.float()).all(), tag
    assert d == 0.0, tag


def _nhwc(x, ld):
    T, H, W, C = x.shape
    out = torch.zeros((T, H, W, ld), dtype=torch.bfloat16, device=x.device)
    out[..., :C] = x.to(torch.bfloat16)
    return out


# ---------------------------------------------------------------------------------------------------- quantize
@pytest.mark.parametrize('src_c', [[5], [32], [544], [32, 64], [256, 256, 32], [5, 70, 13]])
@pytest.mark.parametrize('amax', [0.75, 3.0, 0.0])
def test_quantize_e4m3_static_bit_exact(cuda, src_c, amax):
    from patchfusion_b200 import ops
    T, H, W = 3, 13, 21
    g = _gen('squant', tuple(src_c), amax)
    srcs = []
    for i, c in enumerate(src_c):
        x = torch.randn(T, H, W, c, generator=g, device=cuda) * (1 + i)    # well past the amax: saturation
        x[1, :, :, 0] = -0.0
        x[2, 3, 4, 0] = 1e30                       # far above: 448, not NaN
        ld = fp8_ref.pad_to(c, 8) + (8 if i == 1 else 0)
        s = _nhwc(x, ld)
        if ld > c:
            s[..., c:] = 1e4                       # never read
        srcs.append(s)
    q = torch.full((T, H, W, sum(fp8_ref.pad_to(c, 64) for c in src_c)), 0x7F, dtype=torch.uint8, device=cuda)
    ops.quantize_e4m3_static(srcs, amax, src_c, out=q)
    want = sref.quantize_static_ref(srcs, src_c, amax)
    bad = (q != want).nonzero()
    assert bad.numel() == 0, 'map bytes differ at %s' % bad[:8].tolist()
    assert not torch.isnan(q.view(torch.float8_e4m3fn).float()).any()
    if amax > 0:
        assert (q.view(torch.float8_e4m3fn).float().abs() == 448).any(), 'no saturated value in the probe'
    q1 = ops.quantize_e4m3_static([s[1:2].contiguous() for s in srcs], amax, src_c)
    assert torch.equal(q1[0], q[1])


# ---------------------------------------------------------------------------------------------------- exact conv probes
def _int_operand(shape, g, dev):
    v = torch.randint(-2, 3, shape, generator=g, device=dev).float()
    return v * (torch.rand(shape, generator=g, device=dev) < 0.25)


CASES = [   # (src_c, N, T, H, W): 32 -> BN 32, 64 -> 64, 128 / 256 -> 128, 192 -> 192; partial W / H tiles
    ([5], 32, 3, 37, 29),
    ([32, 64], 64, 2, 16, 8),
    ([256, 256, 32], 128, 2, 19, 23),
    ([64], 192, 3, 17, 9),
    ([32], 256, 1, 8, 16),
    ([256, 256], 256, 9, 64, 96),      # weight-multicast clusters
    ([32], 32, 9, 96, 128),
    ([32], 544, 9, 64, 96),            # last n-tile 160 of 192 columns, 32 pad columns in the e4m3 map
    ([64], 40, 2, 16, 16),             # 24 pad columns inside the 64-column group
    ([32], 160, 2, 24, 40),            # panel padded to 160 rows: BN 64 for the e4m3 output, the last tile half past it
]


@pytest.mark.parametrize('out_kind', ['bf16', 'e4m3'])
@pytest.mark.parametrize('case', CASES, ids=[str(i) for i in range(len(CASES))])
def test_static_conv_exact(cuda, case, out_kind):
    """Integer operands with amax 7 (r = 64, scale 2^-6): every product and sum is exact, so the bf16 output equals the
    fp64 conv rounded once, and the e4m3 output equals the fp64 value quantized at the next ratio (next amax 28: r = 16,
    values past 28 saturate).  The output map is poisoned with 0x7F (an e4m3 NaN) first: its pad columns must be zero."""
    from patchfusion_b200 import ops
    src_c, N, T, H, W = case
    g = _gen('sexact', repr(case))
    xs = []
    for c in src_c:
        x = _int_operand((T, H, W, c), g, cuda)
        x[:, 0, 0, 0] = 7.0
        xs.append(x)
    w = _int_operand((N, sum(src_c), 3, 3), g, cuda)
    w[:, 0, 2, 2] = -7.0
    b = torch.randint(-4, 5, (N,), generator=g, device=cuda).float()
    pw = ops.pack_weight_e4m3(w, b, src_c=src_c)
    q = ops.quantize_e4m3_static([_nhwc(x, fp8_ref.pad_to(c, 8)) for x, c in zip(xs, src_c)], 7.0, src_c)
    ref = F.relu(F.conv2d(torch.cat(xs, -1).permute(0, 3, 1, 2).double(), w.double(), b.double(), padding=1))
    ref = ref.permute(0, 2, 3, 1)
    if out_kind == 'bf16':
        ld = fp8_ref.pad_to(N, 8) + 16
        out = torch.full((T, H, W, ld), 3.0, dtype=torch.bfloat16, device=cuda)
        d = ops.conv3_e4m3_static(pw, q, 7.0, out)
        got, want = out[..., :N].float(), ref.to(torch.bfloat16).float()
        assert (out[..., N:] == 3.0).all(), 'columns past N were written'
    else:
        kc = fp8_ref.pad_to(N, 64)
        out = torch.full((T, H, W, kc + 16), 0x7F, dtype=torch.uint8, device=cuda)
        d = ops.conv3_e4m3_static(pw, q, 7.0, out, next_amax=28.0)
        got = out[..., :kc].view(torch.float8_e4m3fn).float()
        want = torch.zeros_like(got)
        want[..., :N] = sref.quantize(ref.float(), 28.0).float()
        assert (out[..., kc:] == 0x7F).all(), 'bytes past the padded width were written'
        assert not torch.isnan(got).any(), 'an unwritten pad byte'
    bad = (got != want).nonzero()
    assert bad.numel() == 0, '%s block_n %d: %d mismatches, first at %s (got %s want %s)' % (
        out_kind, d.block_n, bad.shape[0], bad[0].tolist(), got[tuple(bad[0])].item(), want[tuple(bad[0])].item())
    print('static exact probe %s src %s N %d T %d %dx%d: block_n %d ok' % (out_kind, src_c, N, T, H, W, d.block_n))


def test_static_conv_refusals(cuda):
    from patchfusion_b200 import lib, ops
    pw = ops.pack_weight_e4m3(torch.randn(64, 32, 3, 3, device=cuda), None)
    q = ops.quantize_e4m3_static([torch.randn(1, 8, 8, 32, device=cuda).bfloat16()], 1.0)
    with pytest.raises((lib.PFError, AssertionError)):      # fp32 output
        ops.conv3_e4m3_static(pw, q, 1.0, torch.zeros((1, 8, 8, 64), dtype=torch.float32, device=cuda))
    with pytest.raises(lib.PFError):                         # e4m3 map narrower than 64 ceil(N / 64)
        ops.conv3_e4m3_static(pw, q, 1.0, torch.zeros((1, 8, 8, 48), dtype=torch.uint8, device=cuda), next_amax=1.0)
    with pytest.raises(lib.PFError):                         # BN 32 with N > 32 and an e4m3 output
        ops.conv3_e4m3_static(pw, q, 1.0, torch.zeros((1, 8, 8, 64), dtype=torch.uint8, device=cuda), next_amax=1.0,
                              block_n=32)


# ---------------------------------------------------------------------------------------------------- models
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
    st = make(fusion_precision='fp8_static')
    lr = st.make_lr(imgs)
    # calibration images that the tests below do not time or compare: seeded, separate
    cal = torch.rand(2, 3, *shape, generator=torch.Generator().manual_seed(7)).to(cuda)
    random.seed(1)
    table = st.calibrate_fp8(st.make_lr(cal), cal, cai_mode='r4', process_num=4)
    return dict(case=case, cfg=cfg, sd=sd, make=make, model=st, imgs=imgs, lr=lr, cal=cal, table=table)


def _infer(model, lr, imgs, seed, **kw):
    random.seed(seed)
    return model(mode='infer', image_lr=lr, image_hr=imgs, **kw)[0].clone()


def test_forward_without_table_refuses(cuda, vits):
    m = vits['make'](fusion_precision='fp8_static')
    with pytest.raises(RuntimeError, match='calibrate_fp8'):
        m(mode='infer', image_lr=vits['lr'][:1], image_hr=vits['imgs'][:1], cai_mode='m1', process_num=2)


def test_calibration_deterministic_and_merges(cuda, vits):
    s = vits
    m = s['make'](fusion_precision='fp8_static')
    a = m.calibrate_fp8(s['lr'][:1], s['imgs'][:1], cai_mode='m1', process_num=2)
    b = m.calibrate_fp8(s['lr'][:1], s['imgs'][:1], cai_mode='m1', process_num=2, reset=True)
    assert a == b and all(v > 0 for v in a.values())
    m.calibrate_fp8(s['lr'][1:2], s['imgs'][1:2], cai_mode='m1', process_num=2)
    merged = dict(m.config['fusion_fp8_amax'])
    both = m.calibrate_fp8(s['lr'][:2], s['imgs'][:2], cai_mode='m1', process_num=2, reset=True)
    assert merged == both
    # the table is what a freshly built model with it runs
    assert {k: float(v) for k, v in m.config['fusion_fp8_amax'].items()} == both


def test_calibration_equals_fp8_tap_amax(cuda, vits):
    """the table is the per-conv maximum over all tiles of the input amax the 'fp8' path computes (its debug taps give
    each conv's bf16 inputs)"""
    s = vits
    f8 = s['make'](fusion_precision='fp8')
    f8.use_cuda_graphs = False
    eng = f8.engine()
    amax = {}
    orig = eng.fusion

    def fusion(*a, **kw):
        taps = {}
        out = orig(*a, taps=taps, **kw)
        convs = {}
        for k, v in taps.items():
            if k.startswith('e4m3.'):
                _, idx, part, _ = k.split('.')
                if part.startswith('src'):
                    convs.setdefault(int(idx), []).append(v.float().abs().max())
        for i, name in enumerate(UNET_ORDER):
            m = torch.stack(convs[i]).max().item()
            amax[name] = max(amax.get(name, 0.0), m)
        return out
    eng.fusion = fusion
    _infer(f8, s['lr'][:1], s['imgs'][:1], 3, cai_mode='m2', process_num=4)
    del eng.fusion
    f8.use_cuda_graphs = True
    random.seed(3)
    table = f8.calibrate_fp8(s['lr'][:1], s['imgs'][:1], cai_mode='m2', process_num=4)
    assert table == amax


def test_model_vs_static_emulation(cuda, vits):
    from oracle import pf_oracle as po
    s = vits
    model, img, lr = s['model'], s['imgs'][:1], s['lr'][:1]
    pn = s['case']['process_num']
    orc = po.Oracle({k: v.to(cuda) for k, v in s['sd'].items()}, s['cfg'])
    bf = s['make']()
    for mode in ('m1', 'm2', 'r4'):
        got = _infer(model, lr, img, 0, cai_mode=mode, process_num=pn)
        with torch.no_grad(), sref.fp8_static_unet(s['table']):
            random.seed(0)
            want = orc.infer(lr, img, cai_mode=mode, process_num=pn).to(got.device).view(got.shape)
        d16 = (got - _infer(bf, lr, img, 0, cai_mode=mode, process_num=pn)).abs()
        err, rng = (got - want).abs().max().item(), (want.max() - want.min()).item()
        print('%s: static FP8 vs static emulation max-abs %.3e (/80 %.3e, /range %.3e); vs bf16 max %.3e mean %.3e'
              % (mode, err, err / MAX_DEPTH, err / rng, d16.max().item(), d16.mean().item()))
        assert torch.isfinite(got).all()
        assert err / MAX_DEPTH < 1e-3, mode


def test_invariances(cuda, vits):
    s = vits
    model, lr, imgs = s['model'], s['lr'], s['imgs']
    _same('static m2 process_num 9 vs 4', _infer(model, lr[:1], imgs[:1], 3, cai_mode='m2', process_num=9),
          _infer(model, lr[:1], imgs[:1], 3, cai_mode='m2', process_num=4))
    for mode in ('m2', 'r4'):
        random.seed(5)
        want = torch.cat([model(mode='infer', image_lr=lr[b:b + 1], image_hr=imgs[b:b + 1], cai_mode=mode,
                                process_num=2)[0].clone() for b in range(imgs.shape[0])])
        _same('static %s B=3 vs 3 x B=1' % mode, _infer(model, lr, imgs, 5, cai_mode=mode, process_num=2), want)
        _same('static %s emulated world 8' % mode,
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
        _same('static mixed geometry image %d' % b, got[b], want[b])


def _count(model, lr, img):
    from patchfusion_b200 import lib
    torch.cuda.synchronize()
    n0 = lib.launch_count()
    y = _infer(model, lr, img, 9, cai_mode='m2', process_num=4)
    torch.cuda.synchronize()
    return y, lib.launch_count() - n0


def test_bf16_and_fp8_unaffected(cuda, vits):
    s = vits
    lr, img = s['lr'][:1], s['imgs'][:1]
    for prec in ('bf16', 'fp8'):
        m = s['make'](fusion_precision=prec)
        _infer(m, lr, img, 9, cai_mode='m2', process_num=4)
        before, n = _count(m, lr, img)
        y8 = _infer(s['model'], lr, img, 9, cai_mode='m2', process_num=4)
        assert not torch.equal(y8, before)
        after, n2 = _count(m, lr, img)
        _same('%s model before / after a static model' % prec, after, before)
        assert n2 == n


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


def test_launch_labels(cuda, vits):
    """per fusion call: 34 static e4m3 convs, 17 static quantize launches, no amax / per-tile quantize launch; with
    PF_OPT_FUSED_RESAMPLE = 1 the 11 fused-resample first convs stay bf16 and their second convs take the quantize"""
    from patchfusion_b200 import lib
    s = vits
    names = _profiled_names(s['model'], s['lr'][:1], s['imgs'][:1])
    calls = names.count('pack_unet_input_kernel')
    n8, nq = names.count('pf_conv3_halo_e4m3_q8_kernel'), names.count('quant_static_kernel')
    print('static m1 forward: %d fusion calls, %d static e4m3 convs, %d static quantize' % (calls, n8, nq))
    assert calls > 0 and n8 == 34 * calls and nq == 17 * calls
    assert names.count('quant_amax_kernel') == 0 and names.count('quant_write_kernel') == 0
    assert names.count('pf_conv3_halo_e4m3_kernel') == 0
    lib.call('pf_set_option', lib.OPT_FUSED_RESAMPLE, 1)
    try:
        names = _profiled_names(s['model'], s['lr'][:1], s['imgs'][:1])
    finally:
        lib.call('pf_set_option', lib.OPT_FUSED_RESAMPLE, 0)
    calls = names.count('pack_unet_input_kernel')
    n8, nq = names.count('pf_conv3_halo_e4m3_q8_kernel'), names.count('quant_static_kernel')
    print('static m1 forward, fused resample: %d calls, %d e4m3 convs, %d quantize' % (calls, n8, nq))
    assert n8 == 23 * calls and nq == 17 * calls
    assert names.count('quant_amax_kernel') == 0 and names.count('quant_write_kernel') == 0


# ---------------------------------------------------------------------------------------------------- vitl stage
def _units(got, ref):
    ulp = torch.pow(2.0, torch.floor(torch.log2(ref.abs().clamp_min(1e-30))) - 7)
    return ((got.double() - ref).abs() / (ulp + ref.abs().max().item() * 2.0 ** -14)).max().item()


def _units8(got, ref):
    """as _units, less half an e4m3 step of ref (the output rounding) per element"""
    step = torch.pow(2.0, torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -6))) - 3)
    ulp = torch.pow(2.0, torch.floor(torch.log2(ref.abs().clamp_min(1e-30))) - 7)
    e = ((got.double() - ref).abs() - 0.5 * step).clamp_min(0)
    return (e / (ulp + ref.abs().max().item() * 2.0 ** -14)).max().item()


@pytest.fixture(scope='module')
def vitl_static(cuda):
    from oracle import pf_oracle as po
    from oracle.make_golden import case_inputs
    from patchfusion_b200.model import PatchFusion
    case = json.load(open(os.path.join(GOLD, 'vitl_tile0.json')))
    cfg, sd, img = case_inputs(case)
    model = PatchFusion(dict(cfg, fusion_precision='fp8_static'))
    model.load_state_dict(sd, strict=True)
    model = model.to(cuda).eval()
    eng = model.engine()
    sdc = {k: v.to(cuda) for k, v in sd.items()}
    orc = po.Oracle(sdc, cfg)
    img = img.to(cuda)
    P = cfg['patch_process_shape']
    H, W = case['image_raw_shape']
    th, tw = case.get('tile', (H // 2, W // 2))
    raw = [(0, 0), (H - th, W - tw)]
    taps = {}
    with torch.no_grad():
        lr = orc.resizer(img)
        crops = torch.cat([orc.resizer(img[:, :, y:y + th, x:x + tw]) for (y, x) in raw])
        fx, fy = 1 / W * P[1], 1 / H * P[0]
        boxes = (torch.tensor([[x, y, x + tw, y + th] for (y, x) in raw], device=cuda).int() *
                 torch.tensor([[fx, fy, fx, fy]], device=cuda)).contiguous()
        cd, cf = eng.branch('coarse', lr.contiguous())
        cd = cd[0].clone()
        cf = [type(f)(f.t.clone(), f.C) for f in cf]
        g2l = eng.g2l(cf)
        cr = crops.contiguous()
        fd, ff = eng.branch('fine', cr)
        eng.calib = {}                                   # calibrate on these two tiles
        eng.fusion(cr, boxes, fd, ff, cd, cf, g2l)
        table = {k: v.item() for k, v in eng.calib.items()}
        eng.calib = None
        eng.set_fp8_amax(table)
        got = eng.fusion(cr, boxes, fd, ff, cd, cf, g2l, taps).clone()
        d_o, f_o = orc.coarse(lr)
        g2l_o = po.g2l_all(sdc, f_o, cfg['guided_fusion'])
        fd_o, ff_o = po.branch_forward(sdc, 'fine_branch.', crops, cfg['fine_branch'])
        rois = [po.roi_crop_zoom(f, boxes, f.shape[-2] / P[0]) for f in f_o]
        droi = po.roi_crop_zoom(d_o, boxes, 1.0)
        with sref.fp8_static_unet(table):
            want = po.fusion_forward(sdc, cfg, fd_o, crops, ff_o, boxes, droi, rois, g2l_o)[:, 0]
        torch.cuda.synchronize()
    return dict(eng=eng, sd=sdc, taps=taps, table=table, got=got, want=want)


def test_vitl_each_static_conv_on_its_own_input(cuda, vitl_static):
    from test_gpu_fp8 import _unet_weights
    s = vitl_static
    Wf, worst = s['eng'].W['fusion'], 0.0
    for name in UNET_ORDER:
        (kin, qin), = [(k, v) for k, v in s['taps'].items() if k.startswith('e4m3s.%s.in.' % name)]
        (kout, out), = [(k, v) for k, v in s['taps'].items() if k.startswith('e4m3s.%s.out.' % name)]
        h, w_ = (int(x) for x in kin.rsplit('.', 1)[1].split('x'))
        pw = Wf[name]
        xq = sref.dequantize(qin.view(torch.float8_e4m3fn), s['table'][name]).double().view(2, h, w_, -1)
        offs = [sum(fp8_ref.pad_to(k, 64) for k in pw.src_c[:i]) for i in range(len(pw.src_c))]
        x = torch.cat([xq[..., o:o + c] for o, c in zip(offs, pw.src_c)], -1).permute(0, 3, 1, 2)
        wt, b, bn = _unet_weights(s['sd'], name)
        wf = wt.float() * bn.view(-1, 1, 1, 1) if bn is not None else wt.float()
        qw, sw = fp8_ref.quantize(wf, fp8_ref.group_amax(wf))
        ref = F.relu(F.conv2d(x, fp8_ref.dequantize(qw, sw).double(), b.double(), padding=1)).permute(0, 2, 3, 1)
        if name.endswith('.0'):
            nxt = name[:-1] + '1'
            got = sref.dequantize(out.view(torch.float8_e4m3fn), s['table'][nxt]).double().view(2, h, w_, -1)
            assert (out.view(2, h, w_, -1)[..., pw.N:] == 0).all(), name
            u = _units8(got[..., :pw.N], ref.clamp(max=s['table'][nxt]))
        else:
            u = _units(out.view(2, h, w_, -1), ref)
        worst = max(worst, u)
        print('%-7s %4dx%-4d -> %3d  worst %.2f units' % (name, h, w_, pw.N, u))
        assert u <= BOUND_UNITS, (name, u)
    print('worst over the 34 static convs: %.2f units' % worst)


def test_vitl_stage_vs_static_emulation(cuda, vitl_static):
    got, want = vitl_static['got'], vitl_static['want']
    assert torch.isfinite(got).all()
    err, rng = (got - want).abs().max().item(), (want.max() - want.min()).item()
    print('vitl_tile0 static fusion vs emulation: max-abs %.3e (/80 %.3e, /range %.3e)' % (err, err / 80, err / rng))
    assert err / MAX_DEPTH < 1e-3
    if not err / rng < RANGE_BAR:
        pytest.xfail('%.1f %% of the output range, above the 2 %% bar (synthetic weights; DESIGN.md section 3)'
                     % (100 * err / rng))
