"""The bf16 stages layer by layer: every GEMM / conv that pf_branch_forward, pf_g2l_forward and pf_fusion_forward issue,
checked on exactly the input it read (its "L.<layer>.<part>" taps) against an fp64 module built from the state dict,
and the glue between layers (LayerNorms, attention, resamples, crops, pooling, the decoder's dataflow) recomputed in
fp64 from the producers' tapped outputs.

Calls (tests/golden fixtures, oracle.make_golden.case_inputs):
  vits_case0   coarse branch B = 1; fine branch on 2 crops; G2L on the coarse maps of 2 images; fusion of 3 tiles with
               tile_image = [1, 0, 1]; the same fusion with PF_OPT_FUSED_RESAMPLE = 1
  vitl_tile0   fine branch and fusion of two 4K tiles (D 1024, features 256)
Per layer the bound is stage_layers_ref.reference's; pure data movement is compared bit for bit, the other glue ops
take the bound of their own kernel test.  Each stage run with taps gives the bits of the run without.
"""
import json
import os

import pytest
import torch
import torch.nn.functional as F

import attn_ref
import bins_ref as br
import stage_layers_ref as sl
import window_ref as wr
from test_gpu_elem import _roi_align_fp64

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(2400)]
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


class _option:
    """set a pf_set_option switch for the duration of a block, restoring the default"""

    def __init__(self, which, value, default=0):
        self.which, self.value, self.default = which, value, default

    def __enter__(self):
        from patchfusion_b200 import lib
        lib.call('pf_set_option', self.which, self.value)

    def __exit__(self, *a):
        from patchfusion_b200 import lib
        lib.call('pf_set_option', self.which, self.default)


def _clone_maps(maps):
    return [type(m)(m.t.clone(), m.C) for m in maps]


def _boxes(eng, H, W, raw, th, tw, dev):
    fx, fy = eng.P[1] / W, eng.P[0] / H
    return (torch.tensor([[x, y, x + tw, y + th] for (y, x) in raw], device=dev).int() *
            torch.tensor([[fx, fy, fx, fy]], device=dev)).contiguous()


def _run(call, fn):
    """fn(taps) -> output tensors; run with and without taps: the same bits (test 4 reads `same`).  Keeps the tapped
    run's outputs as `out`."""
    taps = {}
    with torch.no_grad():
        a = [t.clone() for t in fn(taps)]
        b = [t.clone() for t in fn(None)]
    torch.cuda.synchronize()
    same = all(torch.equal(x.view(torch.uint8) if x.dtype != torch.float32 else x.view(torch.int32),
                           y.view(torch.uint8) if y.dtype != torch.float32 else y.view(torch.int32))
               for x, y in zip(a, b))
    return dict(call=call, taps=taps, same=same, out=a)


def _branch_outs(res):
    """a branch call's outputs: the depth and the six feature maps it returns (the G2L and fusion stages read them)"""
    depth, feats = res
    return [depth] + [f.t for f in feats]


def _build(cuda, name, n_fine, n_coarse, tiles, tile_image, fused=False):
    from oracle import pf_oracle as po
    from oracle.make_golden import case_inputs
    from patchfusion_b200 import lib
    from patchfusion_b200.model import PatchFusion
    case = json.load(open(os.path.join(GOLD, name + '.json')))
    cfg, sd, img0 = case_inputs(case)
    model = PatchFusion(cfg)
    model.load_state_dict(sd, strict=True)
    model = model.to(cuda).eval()
    eng = model.engine()
    H, W = case['image_raw_shape']
    imgs = torch.cat([img0, torch.rand(1, 3, H, W, generator=torch.Generator().manual_seed(11))])[:n_coarse].to(cuda)
    th, tw = H // case['patch_split_num'][0], W // case['patch_split_num'][1]
    lr = po.up(imgs, eng.P).contiguous()

    def crops_of(raw, which):
        return torch.cat([po.up(imgs[b:b + 1, :, y:y + th, x:x + tw], eng.P) for (y, x), b in zip(raw, which)]).contiguous()
    out = dict(cfg=cfg, sd={k: v.to(cuda) for k, v in sd.items()}, eng=eng, P=eng.P, imgs=imgs, runs={})
    with torch.no_grad():
        if n_fine == 2 and not fused and name == 'vits_case0':
            out['runs']['coarse'] = _run('coarse', lambda t: _branch_outs(eng.branch('coarse', lr[:1].contiguous(), t)))
            out['lr1'] = lr[:1]
        cd, cf = eng.branch('coarse', lr, None)
        cd, cf = cd.clone(), _clone_maps(cf)
        out['cf'] = cf
        g2l = _clone_maps(eng.g2l(cf))
        if name == 'vits_case0' and not fused:
            out['runs']['g2l'] = _run('g2l', lambda t: [m.t for m in eng.g2l(cf, t)])
        if n_fine:
            fine2 = crops_of(tiles[:n_fine], tile_image[:n_fine])
            out['runs']['fine'] = _run('fine', lambda t: _branch_outs(eng.branch('fine', fine2, t)))
            out['fine_crops'] = fine2
        crops = crops_of(tiles, tile_image)
        fd, ff = eng.branch('fine', crops, None)
        fd, ff = fd.clone(), _clone_maps(ff)
        boxes = _boxes(eng, H, W, tiles, th, tw, cuda)
        ti = torch.tensor(tile_image, dtype=torch.int32, device=cuda)
        T = len(tiles)

        def fus(t):
            d = torch.zeros((T,) + eng.P, device=cuda)
            return (eng.fusion(crops, boxes, fd, ff, cd, cf, g2l, taps=t, depth_out=d, tile_image=ti),)
        if fused:
            with _option(lib.OPT_FUSED_RESAMPLE, 1):
                out['runs']['fusion'] = _run('fusion', fus)
        else:
            out['runs']['fusion'] = _run('fusion', fus)
        out.update(g2l=g2l, crops=crops, boxes=boxes, tile_image=tile_image, fd=fd, cd=cd, T=T, fused=fused)
    torch.cuda.synchronize()
    return out


@pytest.fixture(scope='module')
def vits(cuda):
    return _build(cuda, 'vits_case0', 2, 2, [(0, 0), (270, 480), (540, 960)], [1, 0, 1])


@pytest.fixture(scope='module')
def vits_fused(cuda):
    return _build(cuda, 'vits_case0', 0, 2, [(0, 0), (270, 480), (540, 960)], [1, 0, 1], fused=True)


@pytest.fixture(scope='module')
def vitl(cuda):
    return _build(cuda, 'vitl_tile0', 2, 1, [(540, 960), (1080, 1920)], [0, 0])


FIXTURES = ['vits', 'vits_fused', 'vitl']


def _calls(request, fx):
    s = request.getfixturevalue(fx)
    return s, [(c, r) for c, r in s['runs'].items()]


def _B(s, call):
    return {'coarse': 1, 'g2l': s['cf'][0].B, 'fine': 2, 'fusion': s['T']}[call]


def _layers(taps):
    """layer names in issue order (first tap of each layer)"""
    out = []
    for k in taps:
        if k.startswith('L.'):
            n = k[2:k.rindex('.')]
            if not out or out[-1] != n:
                assert n not in out, 'layer %s tapped in two places' % n
                out.append(n)
    return out


def _enc_grids(P):
    """the U-Net encoder maps enc[i] the decoder level i reads: inc's at P, down<4-i>'s at P / 2^(5-i)"""
    return {i: (P[0] >> (5 - i), P[1] >> (5 - i)) for i in range(6)}


def _in_grid(s, spec, i, call):
    """the grid source i is read at: a fused-resample conv reads its sources at their own size"""
    key = spec['key']
    if call == 'fusion' and s['fused'] and key[:2] in ('up', 'cv') and key.endswith('.0'):
        lv = int(key[2:-2])
        grids, enc = sl.coarse_map_grids(s['P']), _enc_grids(s['P'])
        if key.startswith('up'):
            return [enc[lv], grids[lv - 1], grids[lv - 1]][i]
        return [enc[0], grids[0]][i] if lv == 0 else grids[lv]
    return spec['in_grid'] or spec['grid']


# ---------------------------------------------------------------------------------------------------- test 1
@pytest.mark.parametrize('fx', FIXTURES)
def test_exact_layer_set(cuda, request, fx):
    s, calls = _calls(request, fx)
    for call, r in calls:
        specs = sl.layer_specs(s['cfg'], call)
        assert _layers(r['taps']) == [sp['key'] for sp in specs], call
        B = _B(s, call)
        for sp in specs:
            t = r['taps']
            k = 'L.%s.' % sp['key']
            for i, c in enumerate(sp['srcs']):
                x = t[k + 'in%d' % i]
                if sp['key'] == 'rs3':
                    assert x.shape[1] == 9 * c
                elif sp['key'] == 'patch':
                    assert x.shape[1] == 592 and (x[:, 588:] == 0).all()
                else:
                    assert x.shape[1] == c, (sp['key'], i, x.shape, c)
                g = _in_grid(s, sp, i, call)
                if sp['key'] != 'rs3':
                    assert x.shape[0] == B * g[0] * g[1], (call, sp['key'], i, x.shape, g)
            assert ('in%d' % len(sp['srcs'])) not in {n[len(k):] for n in t if n.startswith(k)}
            rows = B * sp['grid'][0] * sp['grid'][1]
            if not sp['skip_main']:
                o = t[k + 'out']
                assert o.shape == (rows, 2 * sp['N'] // 3 if sp['vt'] else sp['N']), (sp['key'], o.shape)
            if sp['tail'] is not None:
                assert t[k + 'out3'].shape == (rows, sp['n2'])
        print('%s %s: %d layers' % (fx, call, len(specs)))


# ---------------------------------------------------------------------------------------------------- test 2
def _layer_inputs(s, r, spec, call, B):
    t = r['taps']
    k = 'L.%s.' % spec['key']
    if spec['key'] == 'rs3':
        return [t['L.proj3.out']], False
    ins, rs = [], False
    for i in range(len(spec['srcs'])):
        x = t[k + 'in%d' % i]
        g, (h, w) = spec['grid'], _in_grid(s, spec, i, call)
        if spec['kind'] == 'conv' and spec['in_grid'] is None and (h, w) != g:
            # a fused-resample source at its own size: the reference resamples it in fp64 first
            x = F.interpolate(x.double().view(B, h, w, -1).permute(0, 3, 1, 2), size=g, mode='bilinear',
                              align_corners=True).permute(0, 2, 3, 1).reshape(-1, x.shape[1])
            rs = True
        ins.append(x)
    return ins, rs


def _check_layer(s, r, spec, call, B):
    t = r['taps']
    k = 'L.%s.' % spec['key']
    ins, rs = _layer_inputs(s, r, spec, call, B)
    extra = {p: t[k + p] for p in ('x', 'res1', 'res2') if k + p in t}
    parts = sl.reference(spec, s['sd'], ins, B, extra)
    if rs:      # the resampled operand is stored in bf16 before the MMA: half an ulp of each resampled value
        w, _ = sl.module_weight(spec, s['sd'])
        x = torch.cat([sl._nchw(i, B, spec['grid']) for i in ins], 1).abs()
        extra_b = sl._rows(F.conv2d(x, w.abs(), None, padding=1)) * 2.0 ** -8
        parts = {p: (ref, b + extra_b[:, :ref.shape[1]]) for p, (ref, b) in parts.items()}
    worst = 0.0
    for p, (ref, bound) in parts.items():
        got = t[k + p].double()
        if p == 'vt':
            D = ref.shape[1]
            got = got.view(B, D, -1).transpose(1, 2).reshape(-1, D)
        assert got.shape == ref.shape, (spec['key'], p, got.shape, ref.shape)
        ratio = ((got - ref).abs() / bound)
        assert torch.isfinite(got).all(), (spec['key'], p)
        m = ratio.max().item()
        if m > 1:
            i = int(ratio.argmax())
            print('  %s.%s: worst at %s got %.8g want %.8g bound %.3g' % (
                spec['key'], p, divmod(i, ref.shape[1]), got.flatten()[i].item(), ref.flatten()[i].item(),
                bound.flatten()[i].item()))
        worst = max(worst, m)
    if spec['copy']:        # the ReLU copy is the ReLU of the stored output, bit for bit
        assert torch.equal(t[k + 'out2'], t[k + 'out'].clamp_min(0)), spec['key']
    return worst


@pytest.mark.parametrize('fx', FIXTURES)
def test_each_layer_on_its_own_input(cuda, request, fx):
    s, calls = _calls(request, fx)
    bad = []
    for call, r in calls:
        B = _B(s, call)
        worst = {}
        for spec in sl.layer_specs(s['cfg'], call):
            with torch.no_grad():
                worst[spec['key']] = _check_layer(s, r, spec, call, B)
        top = sorted(worst.items(), key=lambda kv: -kv[1])
        print('%s %s: worst |err| / bound %.3f (%s); %s' % (fx, call, top[0][1], top[0][0],
                                                            ', '.join('%s %.3f' % kv for kv in worst.items())))
        bad += [(call, k, v) for k, v in worst.items() if not v <= 1.0]
    assert not bad, bad


# ---------------------------------------------------------------------------------------------------- test 3
def _ln(x, w, b, eps):
    x = x.double()
    return F.layer_norm(x, (x.shape[-1],), w.double(), b.double(), eps)


def _bf16_check(name, got, ref, slack):
    """|got - ref| <= ulp_bf16(ref) + slack (slack: the fp32 arithmetic of the op, broadcastable)"""
    bound = sl.bf16_ulp(ref) + slack
    r = ((got.double() - ref).abs() / bound).max().item()
    assert r <= 1.0, '%s: %.3f of the bound' % (name, r)
    return r


def _exact(name, got, want):
    assert got.shape == want.shape and torch.equal(got, want), name


def _up(x, B, hw, size):
    """fp64 bilinear align_corners=True of [B*h*w, C] rows to `size` -> rows"""
    t = x.double().view(B, hw[0], hw[1], -1).permute(0, 3, 1, 2)
    if tuple(hw) != tuple(size):
        t = F.interpolate(t, size=tuple(size), mode='bilinear', align_corners=True)
    return t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])


def _glue_branch(s, r, which, B):
    t, sd, cfg = r['taps'], s['sd'], s['cfg']
    from patchfusion_b200.params import branch_hparams
    hp = branch_hparams(cfg[which + '_branch'])
    D, heads, depth = hp['dim'], hp['heads'], hp['depth']
    vit = which + '_branch.core.core.pretrained.'
    g = sl.branch_grids(s['P'])
    gh, gw = g['g']
    seq = gh * gw + 1
    worst = {}
    # tokens (VIT:212-219): patch_im2col normalisation, patch GEMM, cls + bicubic pos from the state dict
    imgs = s['lr1'] if which == 'coarse' else s['fine_crops']
    x = (imgs.double() - torch.tensor(MEAN, device=imgs.device).view(1, 3, 1, 1).double()) / \
        torch.tensor(STD, device=imgs.device).view(1, 3, 1, 1).double()
    cols = F.unfold(x, 14, stride=14).transpose(1, 2).reshape(-1, 588)
    worst['patch_im2col'] = _bf16_check('patch im2col', t['L.patch.in0'][:, :588], cols, 2.0 ** -22 * cols.abs())
    from oracle import pf_oracle as po
    pos = po.interpolated_pos_embed(sd[vit + 'pos_embed'].float(), gh, gw)[0].double()
    pt = t['L.patch.out'].double().view(B, gh * gw, D)
    tok = torch.cat([sd[vit + 'cls_token'].double().view(1, 1, D).expand(B, 1, D), pt], 1) + pos
    err = ((t['tokens'].double().view(B, seq, D) - tok).abs() / (2.0 ** -23 * tok.abs() + 2.0 ** -22 * pos.abs())).max()
    worst['tokens'] = err.item()
    assert err <= 1.0, 'tokens'
    xs = t['tokens']
    for i in range(depth):
        b = vit + 'blocks.%d.' % i
        k = 'L.b%d.' % i
        h1 = _ln(xs, sd[b + 'norm1.weight'], sd[b + 'norm1.bias'], 1e-6)
        worst['norm1'] = max(worst.get('norm1', 0), _bf16_check('b%d norm1' % i, t[k + 'qkv.in0'], h1,
                                                                2.0 ** -18 * (h1.abs() + 1)))
        # attention (scale 1/8) from the qkv's q / k store and its V^T, feeding proj
        qk = t[k + 'qkv.out'].view(B, seq, 2, heads, 64).permute(2, 0, 3, 1, 4)
        v = t[k + 'qkv.vt'].view(B, heads, 64, seq).transpose(-1, -2)
        a = attn_ref.attention_fp64(qk[0], qk[1], v, 0.125).transpose(1, 2).reshape(B * seq, D)
        e = attn_ref.rel_linf(t[k + 'proj.in0'].float(), a.float())
        worst['attention'] = max(worst.get('attention', 0), e / attn_ref.FP64_TOL)
        assert e <= attn_ref.FP64_TOL, 'b%d attention: rel-Linf %.3e' % (i, e)
        _exact('b%d proj x' % i, t[k + 'proj.x'], xs)
        h2 = _ln(t[k + 'proj.out'], sd[b + 'norm2.weight'], sd[b + 'norm2.bias'], 1e-6)
        worst['norm2'] = max(worst.get('norm2', 0), _bf16_check('b%d norm2' % i, t[k + 'fc1.in0'], h2,
                                                                2.0 ** -18 * (h2.abs() + 1)))
        _exact('b%d fc2 in' % i, t[k + 'fc2.in0'], t[k + 'fc1.out'])
        _exact('b%d fc2 x' % i, t[k + 'fc2.x'], t[k + 'proj.out'])
        xs = t[k + 'fc2.out']
        if i >= depth - 4:      # final norm of the last four blocks, cls dropped (DPT:149, VIT:297-321)
            j = i - (depth - 4)
            f = _ln(xs.view(B, seq, D)[:, 1:], sd[vit + 'norm.weight'], sd[vit + 'norm.bias'], 1e-6).reshape(-1, D)
            worst['norm'] = max(worst.get('norm', 0), _bf16_check('proj%d in' % j, t['L.proj%d.in0' % j], f,
                                                                  2.0 ** -18 * (f.abs() + 1)))
    # reassemble: rs0 / rs1 read the projections, layer<i>_rn the reassembled maps
    _exact('rs0 in', t['L.rs0.in0'], t['L.proj0.out'])
    _exact('rs1 in', t['L.rs1.in0'], t['L.proj1.out'])
    for i, src in enumerate(['L.rs0.out', 'L.rs1.out', 'L.proj2.out', 'L.rs3.out']):
        _exact('rn%d in' % i, t['L.rn%d.in0' % i], t[src])
    # the RCUs: conv1 reads the ReLU copy, conv2 adds x (res1) and the path (res2)
    sz = g['sz']
    prev = None
    for wi in (4, 3, 2, 1):
        i = wi - 1
        k = 'L.ff%d.' % wi
        if wi != 4:
            _exact('ff%d u1 c1 in' % wi, t[k + 'u1.c1.in0'], t['L.rn%d.out2' % i])
            _exact('ff%d u1 res1' % wi, t[k + 'u1.c2.res1'], t['L.rn%d.out' % i])
            _exact('ff%d u2 c1 in' % wi, t[k + 'u2.c1.in0'], t[k + 'u1.c2.out2'])
            _exact('ff%d u2 res1' % wi, t[k + 'u2.c2.res1'], t[k + 'u1.c2.out'])
            # FeatureFusionBlock in the reference's order: upsample the previous block's RCU output, THEN out_conv
            # (BLK:147-153), from the tapped input of its out_conv: pins running out_conv at the low resolution
            y = prev
            w, bb = sl.module_weight(dict(mods=[y[0]], bn=None, key='ff'), s['sd'])
            up = sl._nchw(y[1], B, y[2])
            up = F.interpolate(up, size=sz[i], mode='bilinear', align_corners=True)
            ref = sl._rows(F.conv2d(up, w, bb))
            lo = sl._rows(F.conv2d(sl._nchw(y[1], B, y[2]).abs(), w.abs(), bb.abs()))
            ebound = sl.bf16_ulp(_up(lo, B, y[2], sz[i])) + (w.shape[1] + 2) * sl.U * _up(lo, B, y[2], sz[i]) + \
                2.0 ** -22 * lo.abs().max()
            worst['ffb_order'] = max(worst.get('ffb_order', 0),
                                     _bf16_check('ff%d res2 (upsampled out_conv)' % wi, t[k + 'u1.c2.res2'], ref,
                                                 ebound))
        else:
            _exact('ff4 u2 c1 in', t[k + 'u2.c1.in0'], t['L.rn3.out2'])
            _exact('ff4 u2 res1', t[k + 'u2.c2.res1'], t['L.rn3.out'])
        _exact('ff%d out in' % wi, t[k + 'out.in0'], t[k + 'u2.c2.out'])
        prev = ('%s_branch.core.core.depth_head.scratch.refinenet%d.out_conv' % (which, wi), t[k + 'out.in0'], sz[i])
    # the decoder's last resizes: p1 = up(refinenet1 out_conv) feeding output_conv1, its output up to the image
    # feeding output_conv2 (DPT:159-161)
    worst['resize'] = max(_bf16_check('oc1 in (p1)', t['L.oc1.in0'], _up(t['L.ff1.out.out'], B, sz[0], g['p1']),
                                      _roi_slack(t['L.ff1.out.out'], *sz[0])),
                          _bf16_check('oc2.0 in', t['L.oc2.0.in0'], _up(t['L.oc1.out'], B, g['p1'], g['P']),
                                      _roi_slack(t['L.oc1.out'], *g['p1'])))
    _exact('conv2 in', t['L.conv2.in0'], t['L.rn3.out'])
    # the head reads x_d0 = conv2(layer4_rn) and the blocks p4, p3, p2, p1 (PF:198-204, ZD:173-219)
    _exact('seed in', t['L.head.seed_bin_regressor.0.in0'], t['L.conv2.out'])
    _exact('seed_projector in', t['L.head.seed_projector.0.in0'], t['L.conv2.out'])
    for i, src in enumerate(['L.ff3.u1.c2.res2', 'L.ff2.u1.c2.res2', 'L.ff1.u1.c2.res2', 'L.oc1.in0']):
        _exact('projectors.%d in' % i, t['L.head.projectors.%d.0.in0' % i], t[src])
    _exact('clb in0', t['L.head.clb.0.in0'], t['L.oc2.0.out'])
    _exact('clb rel', t['L.head.clb.0.in1'], t['L.oc2.0.out3'].to(torch.bfloat16))
    _glue_head(s, t, B, hp, cfg[which + '_branch'], r['out'][0], 'L.head.clb.0.in2', worst)
    return worst


def _glue_head(s, t, B, hp, bcfg, depth, emb_src, worst):
    """the metric-bins head between its layers (ZD:173-219, PF:297-339) at the bounds of test_gpu_bins_tail.py:
    add_upsampled feeding each attractor MLP, the last embedding resized to the image feeding the log-binomial MLP
    (`emb_src`), and the seed -> four attractors -> log-binomial depth chain, each step from the tapped MLP outputs
    and the previous step's tapped centres.  The fixtures' heads are 'softplus': the seed is the regressor's output."""
    assert hp['bin_centers_type'] == 'softplus'
    P = s['P']
    grid = {sp['key']: sp['grid'] for sp in sl.layer_specs(s['cfg'], 'fusion' if emb_src.endswith('in1') else 'coarse')}
    b_prev = t['L.head.seed_bin_regressor.2.out'].view(B, *grid['head.seed_bin_regressor.2'], -1)
    prev, pg = t['L.head.seed_projector.2.out'], grid['head.seed_projector.2']
    for i in range(4):
        gi = grid['head.projectors.%d.0' % i]
        emb = t['L.head.projectors.%d.2.out' % i]
        e = br.add_upsampled_error(t['L.head.attractors.%d.0.in0' % i].view(B, *gi, -1), emb.view(B, *gi, -1),
                                   prev.view(B, *pg, -1))
        worst['add_upsampled'] = max(worst.get('add_upsampled', 0), e)
        assert e <= 1.0, 'attractors.%d input (add_upsampled): %.3f of the bound' % (i, e)
        ref, _ = br.attractor_fp64(t['L.head.attractors.%d.0.out3' % i].view(B, *gi, -1), hp['n_attractors'][i], b_prev,
                                   hp['attractor_kind'], hp['attractor_type'])
        got = t['b%d' % i].view(B, *gi, -1)
        e, tol = br.rel_linf(got, ref), br.chain_tol(*b_prev.shape[1:3])
        worst['attractor'] = max(worst.get('attractor', 0), e / tol)
        assert e <= tol, 'attractor %d: rel-Linf %.3e > %.3e' % (i, e, tol)
        b_prev, prev, pg = got, emb, gi
    worst['resize'] = max(worst.get('resize', 0), _bf16_check('clb embedding', t[emb_src], _up(prev, B, pg, P),
                                                              _roi_slack(prev, *pg)))
    pt = t['L.head.clb.0.out3'].view(B, *P, -1).cpu()
    temps = (float(bcfg['min_temp']), float(bcfg['max_temp']))
    ref = br.logbinom_depth_fp64(pt, b_prev.cpu(), *P, *temps)
    tol = br.logbinom_tol(br.rel_linf(br.logbinom_depth_oracle32(pt, b_prev.cpu(), *P, *temps), ref))
    e = br.rel_linf(depth.cpu(), ref)
    worst['logbinom'] = e / tol
    assert e <= tol, 'log-binomial depth: rel-Linf %.3e > %.3e' % (e, tol)


def _glue_g2l(s, r, B):
    t, sd = r['taps'], s['sd']
    from patchfusion_b200.params import guided_fusion_hparams
    gf = guided_fusion_hparams(s['cfg']['guided_fusion'], s['P'])
    inv, depth, heads = gf['in_channels'][::-1], gf['depth'][::-1], gf['num_heads'][::-1]
    worst = {}
    for i, (h, w) in enumerate(sl.coarse_map_grids(s['P'])):
        c = inv[i]
        Hp, Wp = wr.padded(h, w)
        g = 'guided_fusion.g2l_list.%d.' % i
        x = s['cf'][i].t[..., :c].double().reshape(B, h * w, c) + sd[g + 'absolute_pos_embed'].double()
        x = x.reshape(-1, c)
        for b in range(depth[i]):
            q = g + 'g2l_layer.blocks.%d.' % b
            k = 'L.g2l%d.b%d.' % (i, b)
            # swin_norm_pad: LN1 (eps 1e-5) on the image, zero rows in the pad
            n1 = torch.zeros(B, Hp, Wp, c, dtype=torch.float64, device=x.device)
            n1[:, :h, :w] = _ln(x, sd[q + 'norm1.weight'], sd[q + 'norm1.bias'], 1e-5).view(B, h, w, c)
            qin = t[k + 'qkv.in0'].view(B, Hp, Wp, c)
            assert (qin[:, h:] == 0).all() and (qin[:, :, w:] == 0).all(), k + 'qkv in: pad rows not zero'
            worst['norm1'] = max(worst.get('norm1', 0), _bf16_check(
                k + 'qkv in', t[k + 'qkv.in0'], n1.view(-1, c), 2.0 ** -18 * (n1.view(-1, c).abs() + 1)))
            # window attention, shifted by 6 in the odd blocks, with the shift mask (SW:325-355)
            a = wr.window_attention_fp64(t[k + 'qkv.out'].view(B, Hp * Wp, 3 * c), sd[q + 'attn.relative_position_bias_table'],
                                         Hp, Wp, c, heads[i], 0 if b % 2 == 0 else wr.WS // 2)
            e = wr.rel_linf(t[k + 'proj.in0'].float().view(B, Hp * Wp, c), a.float())
            worst['window_attention'] = max(worst.get('window_attention', 0), e / wr.FP64_TOL)
            assert e <= wr.FP64_TOL, '%s window attention: rel-Linf %.3e' % (k, e)
            # residual crop: x += proj[:h, :w] (fp32), then LN2 feeding fc1
            pr = t[k + 'proj.out'].double().view(B, Hp, Wp, c)[:, :h, :w].reshape(-1, c)
            xm = x + pr
            got = t[k + 'fc2.x'].double()
            r_ = ((got - xm).abs() / (2.0 ** -23 * xm.abs() + 2.0 ** -22 * (x.abs() + pr.abs()))).max().item()
            worst['residual'] = max(worst.get('residual', 0), r_)
            assert r_ <= 1.0, k + 'residual crop'
            n2 = _ln(got, sd[q + 'norm2.weight'], sd[q + 'norm2.bias'], 1e-5)
            worst['norm2'] = max(worst.get('norm2', 0), _bf16_check(k + 'fc1 in', t[k + 'fc1.in0'], n2,
                                                                    2.0 ** -18 * (n2.abs() + 1)))
            _exact(k + 'fc2 in', t[k + 'fc2.in0'], t[k + 'fc1.out'])
            x = t[k + 'fc2.out'].double()
        # the level's output: the final LayerNorm (eps 1e-5) of the last block's stream (SW:430-432)
        o = _ln(x, sd[g + 'g2l_layer_norm.weight'], sd[g + 'g2l_layer_norm.bias'], 1e-5)
        worst['norm'] = max(worst.get('norm', 0), _bf16_check('g2l%d out' % i, r['out'][i][..., :c].reshape(-1, c), o,
                                                              2.0 ** -18 * (o.abs() + 1)))
    return worst


def _roi_slack(feat, h, w):
    """the fp32 arithmetic of a bilinear sample (crop-zoom or resize) of an h x w map: the weighted sum (2^-22 max |f|)
    and the sample coordinate, rounded in fp32 from a non-dyadic box or scale (a few 2^-24 of a coordinate up to
    max(h, w), times a neighbour difference <= 2 max |f|)"""
    return 2.0 ** -22 * (1 + max(h, w)) * feat.float().abs().max().item()


def _glue_fusion(s, r, T):
    t = r['taps']
    P = s['P']
    from patchfusion_b200.params import guided_fusion_hparams
    gf = guided_fusion_hparams(s['cfg']['guided_fusion'], P)
    inv = gf['in_channels'][::-1]
    grids = sl.coarse_map_grids(P)
    images = s['tile_image']
    boxes = s['boxes'].cpu()
    worst = {}
    # ROI crop-zoom of the coarse maps at each level's scale, from image tile_image[t] (PF:240-257)
    for i in range(5):
        f = s['cf'][i]
        h, w = grids[i]
        ref = _roi_align_fp64(f.t[..., :f.C].cpu(), boxes, h / P[0], images).to(t['L.fc0.in0'].device)
        ref = ref.reshape(-1, f.C)
        worst['roi'] = max(worst.get('roi', 0), _bf16_check('fc%d roi' % i, t['L.fc%d.in0' % i], ref,
                                                            _roi_slack(f.t, h, w)))
    # pack_unet_input: [coarse depth ROI, fine depth, crop RGB] (PF:259-267, GF:179), the depth ROI from image
    # tile_image[t] at scale 1; the fine depth and the crops are only moved (rounded to bf16)
    H, W = P
    u = t['L.inc.0.in0'].view(T, H, W, 5)
    _exact('unet input fine depth', u[..., 1], s['fd'].to(torch.bfloat16))
    _exact('unet input rgb', u[..., 2:], s['crops'].permute(0, 2, 3, 1).to(torch.bfloat16))
    ref = _roi_align_fp64(s['cd'].unsqueeze(-1).cpu(), boxes, 1.0, images)[..., 0].to(u.device)
    worst['roi'] = max(worst['roi'], _bf16_check('unet input coarse depth', u[..., 0], ref, _roi_slack(s['cd'], H, W)))
    # maxpool, and which decoder level reads which encoder map
    enc = {5: 'L.inc.1.out'}
    for i in range(5):
        src = 'L.inc.1.out' if i == 0 else 'L.down%d.1.out' % (i - 1)
        hw = P if i == 0 else (P[0] >> i, P[1] >> i)
        x = t[src].view(T, hw[0], hw[1], -1)
        want = x[:, :hw[0] // 2 * 2, :hw[1] // 2 * 2].float().view(T, hw[0] // 2, 2, hw[1] // 2, 2, -1)
        want = want.amax(dim=(2, 4)).to(torch.bfloat16).reshape(-1, x.shape[-1])
        _exact('down%d maxpool' % i, t['L.down%d.0.in0' % i], want)
        _exact('down%d.1 in' % i, t['L.down%d.1.in0' % i], t['L.down%d.0.out' % i])
        enc[4 - i] = 'L.down%d.1.out' % i
    _exact('inc.1 in', t['L.inc.1.in0'], t['L.inc.0.out'])
    enc_hw = _enc_grids(P)
    fused = s['fused']
    for i in range(6):
        g = grids[i]
        if i > 0:
            srcs = [('up%d.0' % i, 0, (enc[i], enc_hw[i])), ('up%d.0' % i, 1, ('L.cv%d.1.out' % (i - 1), grids[i - 1])),
                    ('up%d.0' % i, 2, ('L.fc%d.out' % (i - 1), grids[i - 1])),
                    ('cv%d.0' % i, 0, ('L.up%d.1.out' % i, g))]
        else:
            srcs = [('cv0.0', 0, (enc[0], enc_hw[0]))]
        for layer, j, src in srcs:
            got = t['L.%s.in%d' % (layer, j)]
            x = t[src[0]]
            if fused or tuple(src[1]) == tuple(g):
                _exact('%s in%d' % (layer, j), got, x)
            else:
                ref = _up(x, T, src[1], g)
                worst['resize'] = max(worst.get('resize', 0), _bf16_check(
                    '%s in%d' % (layer, j), got, ref, _roi_slack(x, *src[1])))
        _exact('up/cv%d.1 in' % i, t['L.cv%d.1.in0' % i], t['L.cv%d.0.out' % i])
        if i > 0:
            _exact('up%d.1 in' % i, t['L.up%d.1.in0' % i], t['L.up%d.0.out' % i])
        # the G2L map cropped at this level's scale from image tile_image[t]
        gm = s['g2l'][i]
        ref = _roi_align_fp64(gm.t[..., :gm.C].cpu(), boxes, g[0] / P[0], images).to(got.device).reshape(-1, gm.C)
        worst['roi'] = max(worst.get('roi', 0), _bf16_check('cv%d roi' % i, t['L.cv%d.0.in1' % i], ref,
                                                            _roi_slack(gm.t, g[0], g[1])))
    _exact('head seed in', t['L.head.seed_bin_regressor.0.in0'], t['L.cv0.1.out'])
    _exact('head seed_projector in', t['L.head.seed_projector.0.in0'], t['L.cv0.1.out'])
    _exact('clb in0', t['L.head.clb.0.in0'], t['L.cv5.1.out'])
    for i in range(4):
        _exact('projectors.%d in' % i, t['L.head.projectors.%d.0.in0' % i], t['L.cv%d.1.out' % (i + 1)])
    from patchfusion_b200.params import branch_hparams
    _glue_head(s, t, T, branch_hparams(s['cfg']['coarse_branch']), s['cfg']['coarse_branch'], r['out'][0],
               'L.head.clb.0.in1', worst)
    return worst


@pytest.mark.parametrize('fx', FIXTURES)
def test_glue_between_layers(cuda, request, fx):
    s, calls = _calls(request, fx)
    for call, r in calls:
        with torch.no_grad():
            if call in ('coarse', 'fine'):
                w = _glue_branch(s, r, call, _B(s, call))
            elif call == 'g2l':
                w = _glue_g2l(s, r, _B(s, call))
            else:
                w = _glue_fusion(s, r, s['T'])
        print('%s %s glue, worst / bound: %s' % (fx, call, ', '.join('%s %.3f' % kv for kv in w.items())))


# ---------------------------------------------------------------------------------------------------- test 4
@pytest.mark.parametrize('fx', FIXTURES)
def test_taps_do_not_perturb(cuda, request, fx):
    s, calls = _calls(request, fx)
    for call, r in calls:
        assert r['same'], '%s %s: output bits differ with taps' % (fx, call)
        assert any(k.startswith('L.') for k in r['taps'])
