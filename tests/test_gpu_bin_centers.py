"""The normed / hybrid bin-centre heads on the GPU.

Kernels: pf_seed_bins and pf_attractor_normed against the fp64 references and the fp32 emulations of
tests/bin_centers_ref.py, at every level of the head's resize chain (nA 16/8/4/1) and the edge shapes of
test_gpu_bins_tail.py, on bin centres that need the sort (reversed, interleaved, ties, all equal) and the clip
(outside [0, 1]); NaN where the kernels must not read, a sentinel after every output, >= 3 grid-stride passes, and
two runs bit-identical.

Model: a vits PatchFusion per case of oracle/make_golden_bin_centers.py (normed, hybrid1, hybrid2, coarse normed with
fine softplus) against the reference fixture and the oracle executed by torch on the GPU; each case's depth tolerance
is one that the other cases' outputs miss by >= 4x.  BaselinePretrain's coarse and fine targets with normed branches;
a normed PatchFusion with B = 2 and emulated W = 2 sharding, bit for bit."""
import os
import random

import numpy as np
import pytest
import torch

import bin_centers_ref as cr
import bins_ref as br

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
GOLD = os.path.join(os.path.dirname(__file__), 'golden')


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _passes(total):
    per_pass = 64 * _sms()          # eight 256-thread blocks per SM, one warp per pixel
    n = (total + per_pass - 1) // per_pass
    print('%d pixels, %d passes of %d' % (total, n, per_pass))
    return n


def _out(n, cuda):
    return torch.full((n + 64,), br.SENTINEL, device=cuda)


def _nan_tail(x, cuda):
    B, h, w, C = x.shape
    buf = torch.full((x.numel() + (w + 1) * C,), float('nan'), device=cuda)
    buf[:x.numel()] = x.reshape(-1).to(cuda)
    return buf


def _untouched(buf, n, tag):
    assert (buf[n:] == br.SENTINEL).all(), tag + ': the kernel wrote past its output'


# ------------------------------------------------------------------------------------------------------ pf_seed_bins
@pytest.mark.parametrize('rng', [(1e-3, 80.0), (0.05, 40.0)], ids=['1e-3..80', '0.05..40'])
@pytest.mark.parametrize('flags', [1, 2, 3], ids=['normed', 'unit', 'normed+unit'])
def test_seed_bins(cuda, flags, rng):
    from patchfusion_b200 import ops
    lo, hi = rng
    gen = torch.Generator().manual_seed(10 + flags)
    P = 3 * 101 * 97
    assert _passes(P) >= 3 and P % (64 * _sms())
    S = cr.seed_case(P, gen, ld=72)
    Sd = S.to(cuda)
    n = P * br.NBINS

    def run():
        out = _out(n, cuda)
        ops.seed_bins(Sd, br.NBINS, flags, lo, hi, out)
        return out

    a, b = run(), run()
    torch.cuda.synchronize()
    assert torch.equal(a, b), 'two runs differ'
    _untouched(a, n, 'seed_bins')
    got = a[:n].view(P, br.NBINS).cpu()
    ref, scale = cr.seed_bins_fp64(S, lo, hi, flags & 1, flags & 2)
    e64 = cr.seed_error(got, ref, scale)
    emu = cr.seed_bins_emulated(S, lo, hi, flags).double()
    e_emu = cr.seed_error(got, emu, scale)
    print('flags %d range %s: vs fp64 %.2f of the bound, vs emulation %.2f' % (flags, rng, e64 / cr.SEED_TOL,
                                                                                 e_emu / cr.SEED_TOL))
    assert e64 <= cr.SEED_TOL and e_emu <= cr.SEED_TOL


# ------------------------------------------------------------------------------------------------ pf_attractor_normed
def _attractor(A, nA, b_prev, flags, lo, hi, cuda):
    from patchfusion_b200 import ops
    B, H, W, _ = A.shape
    n = B * H * W * br.NBINS
    Ad, bp = A.to(cuda), _nan_tail(b_prev, cuda)
    bpv = bp[:b_prev.numel()].view(b_prev.shape)

    def run():
        b, c = _out(n, cuda), _out(n, cuda)
        ops.attractor_normed(Ad, nA, bpv, flags, lo, hi, b[:n].view(B, H, W, -1), c[:n].view(B, H, W, -1))
        return b, c

    (b1, c1), (b2, c2) = run(), run()
    torch.cuda.synchronize()
    assert torch.equal(b1, b2) and torch.equal(c1, c2), 'two runs differ'
    _untouched(b1, n, 'b_new')
    _untouched(c1, n, 'centres')
    return b1[:n].view(B, H, W, -1).cpu(), c1[:n].view(B, H, W, -1).cpu()


def _check(tag, A2, A, nA, b_prev, lo, hi, cuda):
    hw = b_prev.shape[1:3]
    for flags in range(4):
        kind, typ = br.ATTRACTOR_FLAGS[flags]
        b, c = _attractor(A, nA, b_prev, flags, lo, hi, cuda)
        b64, c64, _ = cr.attractor_normed_fp64(A2, nA, b_prev, lo, hi, kind, typ)
        be, ce = cr.attractor_normed_emulated(A2, nA, b_prev, flags, lo, hi)
        e64 = cr.attractor_errors(b, c, b64, c64, lo, hi, hw, nA, kind)
        eem = cr.attractor_errors(b, c, be.double(), ce.double(), lo, hi, hw, nA, kind)
        print('%s flags %d nA %d: b %.2f / centres %.2f of the bound vs fp64, %.2f / %.2f vs emulation' %
              (tag, flags, nA, *e64, *eem))
        assert max(e64) <= 1 and max(eem) <= 1, (tag, flags)


@pytest.mark.parametrize('order', cr.ORDERS)
@pytest.mark.parametrize('level', range(4))
def test_attractor_normed_chain(cuda, level, order):
    hw, HW, nA = br.CHAIN[level]
    gen = torch.Generator().manual_seed(500 + 10 * level + cr.ORDERS.index(order))
    B = 2 if level < 3 else 1
    if level >= 2:
        assert _passes(B * HW[0] * HW[1]) >= 3
    A2, A, b_prev = cr.attractor_normed_case(B, hw, HW, nA, gen, order)
    _check('chain %dx%d->%dx%d %s' % (*hw, *HW, order), A2, A, nA, b_prev, 1e-3, 80.0, cuda)


@pytest.mark.parametrize('hw,HW', [((28, 37), (28, 37)), ((1, 19), (28, 37)), ((1, 1), (7, 9)), ((13, 19), (61, 83))],
                         ids=['same-size', 'one-row-source', 'one-pixel-source', '13x19-61x83'])
def test_attractor_normed_edges(cuda, hw, HW):
    gen = torch.Generator().manual_seed(600 + HW[0])
    for nA in (16, 3):
        for order in ('outside', 'reversed'):
            A2, A, b_prev = cr.attractor_normed_case(3, hw, HW, nA, gen, order)
            _check('edge %dx%d->%dx%d %s' % (*hw, *HW, order), A2, A, nA, b_prev, 0.05, 40.0, cuda)


# ------------------------------------------------------------------------------------------------------ model level
def _gold(name):
    return dict(np.load(os.path.join(GOLD, 'bin_centers_%s.npz' % name)))


def _model(name, cuda):
    from oracle.make_golden_bin_centers import case_inputs
    from patchfusion_b200.model import PatchFusion
    cfg, sd, img = case_inputs(name)
    m = PatchFusion(cfg)
    m.load_state_dict(sd, strict=True)
    return cfg, sd, img, m.to(cuda).eval()


DEPTH_TOL = 1e-2            # BaselinePretrain with normed branches: TOL of the normed case
CENTER_TOL = 5e-2           # final bin centres / max_depth (tests/test_gpu_model.py: 3e-2 of the softplus taps)


def _depth_err(got, want, max_depth):
    got, want = torch.as_tensor(got).float().cpu(), torch.as_tensor(want).float().cpu()
    assert got.shape == want.shape and torch.isfinite(got).all()
    return (got - want).abs().max().item() / max_depth


@pytest.fixture(scope='module')
def cases(cuda):
    """every case's GPU outputs at the fixture's sample points"""
    from oracle import bin_centers_oracle as bco
    from oracle import pf_oracle as po
    from oracle.make_golden_bin_centers import CASES, MODEL
    st, sc, cc = MODEL['sample_stride'], MODEL['infer_stride'], MODEL['center_channels']
    res = {}
    for name in CASES:
        cfg, sd, img, model = _model(name, cuda)
        eng = model.engine()
        lr = model.resizer(img.to(cuda))
        taps = {}
        cd, cf = eng.branch('coarse', lr.contiguous(), taps)
        ct, ft = CASES[name]
        key = lambda t: 'centers' if t in ('normed', 'hybrid2') else 'b3'               # noqa: E731
        out = dict(coarse_depth=cd[:, None, ::st, ::st].cpu().clone(),
                   coarse_centers=taps[key(ct)].permute(0, 3, 1, 2)[:, ::cc, ::st, ::st].cpu().clone())
        cd = cd[0].clone()
        cf = [type(f)(f.t.clone(), f.C) for f in cf]
        g2l = eng.g2l(cf)
        H, W = MODEL['image_raw_shape']
        h, w = H // 2, W // 2
        raw = [(0, 0), (h // 2, w // 2)]
        P = cfg['patch_process_shape']
        fx, fy = 1 / W * P[1], 1 / H * P[0]
        boxes = torch.tensor([[x, y, x + w, y + h] for (y, x) in raw]).int() * torch.tensor([[fx, fy, fx, fy]])
        crops = torch.cat([model.resizer(img[:, :, y:y + h, x:x + w].to(cuda)) for (y, x) in raw]).contiguous()
        taps = {}
        fd, ff = eng.branch('fine', crops, taps)
        out['fine_depth'] = fd[:, None, ::st, ::st].cpu().clone()
        out['fine_centers'] = taps[key(ft)].permute(0, 3, 1, 2)[:, ::cc, ::st, ::st].cpu().clone()
        taps = {}
        fu = eng.fusion(crops, boxes.to(cuda).contiguous(), fd, ff, cd, cf, g2l, taps)
        torch.cuda.synchronize()
        out['fusion_depth'] = fu[:, None, ::st, ::st].cpu().clone()
        fc = taps[key(ct)].view(2, *g2l[4].hw, -1).permute(0, 3, 1, 2)      # the fusion head's last block
        out['fusion_centers'] = fc[:, ::cc, ::st, ::st].cpu().clone()
        # the oracle executed by torch on the GPU (fp32, TF32 off) on the same inputs
        sdc = {k: v.to(cuda) for k, v in sd.items()}
        with torch.no_grad(), bco.typed_heads(cfg):
            d_o, f_o = po.branch_forward(sdc, 'coarse_branch.', lr, cfg['coarse_branch'])
            fd_o, ff_o = po.branch_forward(sdc, 'fine_branch.', crops, cfg['fine_branch'])
            bx = boxes.to(cuda)
            rois = [po.roi_crop_zoom(f, bx, f.shape[-2] / P[0]) for f in f_o]
            g2l_o = po.g2l_all(sdc, f_o, cfg['guided_fusion'])
            fu_o = po.fusion_forward(sdc, cfg, fd_o, crops, ff_o, bx, po.roi_crop_zoom(d_o, bx, 1.0), rois, g2l_o)
        out['oracle'] = dict(coarse_depth=d_o[..., ::st, ::st].cpu(), fine_depth=fd_o[..., ::st, ::st].cpu(),
                             fusion_depth=fu_o[..., ::st, ::st].cpu())
        random.seed(0)
        y, _ = model(mode='infer', image_lr=lr, image_hr=img.to(cuda), cai_mode='m1', process_num=MODEL['process_num'])
        out['infer_m1'] = y[..., ::sc, ::sc].cpu().clone()
        out['cfg'] = cfg
        res[name] = out
        del model, eng, sdc
        torch.cuda.empty_cache()
    return res


HEADS = {'coarse': 'coarse', 'fine': 'fine', 'fusion': 'top', 'infer_m1': 'top'}


def _max_depth(cfg, head):
    return float(cfg['max_depth'] if HEADS[head] == 'top' else cfg[head + '_branch']['max_depth'])


# Depth tolerance per (case, head), as max |d - d_ref| / the head's max_depth ('fusion' also bounds the stitched m1
# output).  A head with normed attractors works on centres normalised to [0, 1], where the attractors act over
# ~1/sqrt(300) = 0.06: the bf16 activations of the attractor MLP move them by ~1e-2, and the metric output scales that
# by (max - min); a normed seed's widths carry the same relative error.  Measured on an H100 80GB HBM3 (GPU result
# against the fixture, max over the sampled points): 4e-3 - 1.3e-2 for the branch heads, 9e-3 - 2.4e-2 for the
# fusion head and the stitched output.  The softplus head's attractors act on metric centres metres apart and barely move them, so
# its bf16 error stays at tests/test_gpu_model.py's 1e-3 (3e-5 measured).  Each value is also >= 4x below the
# distance to every other case's output (8x - 1000x measured), which shows the configured type reaches the kernels.
TOL = {('normed', 'coarse'): 1e-2, ('normed', 'fine'): 1e-2, ('normed', 'fusion'): 2e-2,
       ('hybrid1', 'coarse'): 1e-2, ('hybrid1', 'fine'): 1e-2, ('hybrid1', 'fusion'): 2e-2,
       ('hybrid2', 'coarse'): 2e-2, ('hybrid2', 'fine'): 2e-2, ('hybrid2', 'fusion'): 4e-2,
       ('mixed', 'coarse'): 1e-2, ('mixed', 'fine'): 1e-3, ('mixed', 'fusion'): 2e-2}


@pytest.mark.parametrize('name', ['normed', 'hybrid1', 'hybrid2', 'mixed'])
def test_patchfusion_against_fixture_and_oracle(cuda, cases, name):
    out, cfg = cases[name], cases[name]['cfg']
    g = _gold(name)
    p = name + '_'
    bad = []
    for head in ('coarse', 'fine', 'fusion', 'infer_m1'):
        md = _max_depth(cfg, head)
        tol = TOL[(name, 'fusion' if head == 'infer_m1' else head)]
        dk = head if head == 'infer_m1' else head + '_depth'
        e_fix = _depth_err(out[dk], g[p + dk], md)
        e_orc = _depth_err(out[dk], out['oracle'][dk], md) if dk in out['oracle'] else 0.0
        msg = '%s %s depth: vs fixture %.3e, vs GPU oracle %.3e (tol %.0e)' % (name, head, e_fix, e_orc, tol)
        if head != 'infer_m1':
            e_cen = _depth_err(out[head + '_centers'], g[p + head + '_centers'], md)
            msg += '; final centres vs fixture %.3e (tol %.0e)' % (e_cen, CENTER_TOL)
            if not e_cen < CENTER_TOL:
                bad.append((head, 'centres', e_cen))
        print(msg)
        if not max(e_fix, e_orc) < tol:
            bad.append((head, 'depth', e_fix, e_orc))
        # the same tolerance must separate this case from the others: the config reaches the kernels
        for other in cases:
            # 'mixed' and 'normed' share the coarse branch (same type, same weights): nothing to tell apart there
            if other == name or (head == 'coarse' and CASE_TYPES[other][0] == CASE_TYPES[name][0]):
                continue
            e_x = _depth_err(out[dk], _gold(other)[other + '_' + dk], md)
            print('   vs the %s fixture: %.3e (%.0fx the tolerance)' % (other, e_x, e_x / tol))
            if not e_x >= 4 * tol:
                bad.append((head, other, e_x))
    assert not bad, bad


CASE_TYPES = {'normed': ('normed', 'normed'), 'hybrid1': ('hybrid1', 'hybrid1'), 'hybrid2': ('hybrid2', 'hybrid2'),
              'mixed': ('normed', 'softplus')}


def test_patchfusion_batch_and_sharding_normed(cuda):
    """B = 2 equals two B = 1 calls, and emulated W = 2 tile sharding equals the unsharded run, bit for bit"""
    from oracle.make_golden_bin_centers import MODEL
    cfg, sd, img, model = _model('normed', cuda)
    img2 = torch.rand(1, 3, *MODEL['image_raw_shape'], generator=torch.Generator().manual_seed(77))
    imgs = torch.cat([img, img2]).to(cuda)
    lr = model.make_lr(imgs)
    for mode in ('m1', 'r4'):
        random.seed(5)
        seq = torch.cat([model(mode='infer', image_lr=lr[b:b + 1], image_hr=imgs[b:b + 1], cai_mode=mode,
                               process_num=2)[0].clone() for b in range(2)])
        random.seed(5)
        bat = model(mode='infer', image_lr=lr, image_hr=imgs, cai_mode=mode, process_num=2)[0].clone()
        random.seed(5)
        sh = model(mode='infer', image_lr=lr, image_hr=imgs, cai_mode=mode, process_num=2, shard=('emulate', 2))[0].clone()
        assert torch.isfinite(bat).all()
        d1, d2 = (bat - seq).abs().max().item(), (sh - bat).abs().max().item()
        print('%s: B=2 vs 2 x B=1 %.3e, emulated W=2 vs unsharded %.3e' % (mode, d1, d2))
        assert d1 == 0.0 and d2 == 0.0


@pytest.mark.parametrize('target', ['coarse', 'fine'])
def test_baseline_pretrain_normed(cuda, target):
    """BaselinePretrain with a normed branch (the fixture's normed case weights) against BaselineOracle on the GPU"""
    from oracle import bin_centers_oracle as bco
    from oracle.baseline_oracle import BaselineOracle
    from oracle.make_golden_bin_centers import RANGES, case_inputs
    from patchfusion_b200.baseline import BaselinePretrain
    from test_baseline_host import pretrain_model_cfg
    _, sd, img = case_inputs('normed')
    kw = dict(image_raw_shape=(1080, 1920), patch_split_num=(2, 2)) if target == 'fine' else {}
    cfg = pretrain_model_cfg('vits', target, **kw)
    for b in ('coarse', 'fine'):
        cfg[b + '_branch']['bin_centers_type'] = 'normed'
        cfg[b + '_branch']['min_depth'], cfg[b + '_branch']['max_depth'] = RANGES[b]
    cfg.pop('type')
    m = BaselinePretrain(**cfg)
    pre = target + '_branch.'
    m.load_dict({k[len(pre):]: v for k, v in sd.items() if k.startswith(pre)})
    m = m.to(cuda).eval()
    sdc = {k: v.to(cuda) for k, v in sd.items()}
    orc = BaselineOracle(sdc, cfg, target)
    img = img.to(cuda)
    md = RANGES[target][1]
    if target == 'coarse':
        import torch.nn.functional as F
        lr = F.interpolate(img, (392, 518), mode='bilinear', align_corners=True)
        y, _ = m(mode='infer', image_lr=lr, image_hr=None)
        with torch.no_grad(), bco.typed_heads(cfg):
            want = orc.infer(lr, None)
    else:
        random.seed(0)
        y, _ = m(mode='infer', image_lr=None, image_hr=img, cai_mode='m1', process_num=2)
        random.seed(0)
        with torch.no_grad(), bco.typed_heads(cfg):
            want = orc.infer(None, img, cai_mode='m1', process_num=2)
    e = _depth_err(y, want, md)
    print('BaselinePretrain %s normed vs oracle: %.3e of max_depth' % (target, e))
    assert e < DEPTH_TOL
