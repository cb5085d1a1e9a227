"""pf_window_attention (window_attention_kernel) against two references (tests/window_ref.py), at the G2L levels' real
geometries, every compiled head dim, the grid edges and adversarial softmax inputs, plus the batched Swin helpers and
one Swin block through the ops wrappers:

  fp64       the reference's formulation in fp64 on the bf16 qkv: global rel-L-inf <= FP64_TOL (8e-3).
  emulated   the kernel's own fp32 algorithm: every element within one bf16 ulp of |emulated| plus EMU_ABS x max |V|.

Every qkv buffer is followed by NaN rows and every output by sentinel rows: the NaN must not reach the result and the
sentinel must survive.  Each case runs twice and must give the same bits.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

import window_ref as wr

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

# the six G2L levels of the default (vitl) model, high to low resolution: (H, W, C, heads)
LEVELS = [(392, 518, 32, 8), (224, 296, 256, 8), (112, 148, 256, 16), (56, 74, 256, 16), (28, 37, 256, 32),
          (14, 19, 256, 32)]
EXTRA = 5                       # NaN rows after the last image's qkv, sentinel rows after the output
BF16 = torch.bfloat16
# Swin block chain, attention update against fp64 from the block's input: on top of the attention output's own bf16
# store (what FP64_TOL covers) the update inherits two more bf16 stores, the LayerNorm output and qkv, where the
# kernels' fp32 values and the fp64 ones can round to neighbouring bf16 values.  Each flip moves the update by about
# as much as a flip of the attention output, so twice FP64_TOL.  Measured on an H100: at most 8.2e-3 (392 x 518,
# C 32, B 2), where with 4-dim heads and a 32-wide projection a few flips are not averaged out.
CHAIN_TOL = 2 * wr.FP64_TOL


def _ops():
    from patchfusion_b200 import ops
    return ops


def launch(qkv, table, Hp, Wp, C, heads, shift):
    """qkv [B, Hp * Wp, 3C] fp32 (bf16 values) -> the kernel's output [B, Hp * Wp, C] bf16 through
    pf_window_attention_batched, with NaN rows after qkv and sentinel rows after the output"""
    ops = _ops()
    B, n = qkv.shape[0], qkv.shape[0] * Hp * Wp
    qb = torch.full((n + EXTRA, 3 * C), float('nan'), dtype=BF16, device='cuda')
    qb[:n] = qkv.reshape(n, 3 * C)
    out = torch.full((n + EXTRA, C), wr.SENTINEL, dtype=BF16, device='cuda')
    ops.call('pf_window_attention_batched', qb, table.cuda().contiguous(), B, Hp, Wp, C, heads, shift, out,
             ops.stream_ptr())
    torch.cuda.synchronize()
    assert (out[n:] == wr.SENTINEL).all(), 'the kernel wrote past the last image'
    return out[:n].view(B, Hp * Wp, C)


def run_case(tag, qkv, table, H, W, C, heads, shift, emulate=True):
    """launch twice (same bits), check against fp64 and the emulation; -> (output, fp64 error, emulation error)"""
    Hp, Wp = wr.padded(H, W)
    qkv, table = qkv.cuda(), table.cuda()
    got = launch(qkv, table, Hp, Wp, C, heads, shift)
    again = launch(qkv, table, Hp, Wp, C, heads, shift)
    assert torch.equal(got, again), tag + ': two launches differ'
    e64 = wr.rel_linf(got, wr.window_attention_fp64(qkv, table, Hp, Wp, C, heads, shift))
    eemu = None
    if emulate:
        eemu = wr.emu_error(got, wr.window_attention_emulated(qkv, table, Hp, Wp, C, heads, shift), qkv, C)
    print('%-44s fp64 %.2e (%.2f of bound)  emulation %s' % (
        tag, e64, e64 / wr.FP64_TOL, '-' if eemu is None else '%.2f of bound' % eemu))
    assert e64 <= wr.FP64_TOL, '%s: rel-Linf %.3e against fp64' % (tag, e64)
    assert eemu is None or eemu <= 1.0, '%s: %.2f x the emulation bound' % (tag, eemu)
    return got, e64, eemu


# ------------------------------------------------------------------------------------------------ real levels
def test_levels_are_the_engines(cuda):
    """LEVELS is what the default model's G2L stage runs (engine order is low to high resolution)"""
    from patchfusion_b200.configs import depth_anything_patchfusion
    from patchfusion_b200.engine import Engine
    from patchfusion_b200.params import guided_fusion_hparams, state_layout
    cfg = depth_anything_patchfusion('vitl')
    gf = guided_fusion_hparams(cfg['guided_fusion'], cfg['patch_process_shape'])
    assert [(c, h, n) for c, h, n in zip(gf['in_channels'], gf['num_heads'], gf['num_patches'])] == \
        [(C, h, H * W) for H, W, C, h in LEVELS]
    sd = {k: torch.zeros(shape, dtype=dt) for k, (shape, dt, _) in state_layout(cfg).items()
          if not k.startswith(('coarse_branch.', 'fine_branch.'))}
    eng = Engine(cfg, sd, cuda, parts=('fusion',))
    assert [(g.C, g.heads, g.ape_rows) for g in eng.c_fusion.g2l] == [(C, h, H * W) for H, W, C, h in LEVELS[::-1]]


@pytest.mark.parametrize('shift', [0, 6])
@pytest.mark.parametrize('level', range(6))
def test_level(cuda, level, shift):
    H, W, C, heads = LEVELS[level]
    qkv, table = wr.make_case('random', 1, H, W, C, heads, shift, seed=level)
    run_case('level %d %dx%d C%d h%d shift %d' % (level, H, W, C, heads, shift), qkv, table, H, W, C, heads, shift)


@pytest.mark.parametrize('shift', [0, 6])
@pytest.mark.parametrize('hd', [2, 4, 8, 16, 32])
def test_head_dim(cuda, hd, shift):
    """every compiled instantiation, HD = 2 included (no shipped config uses it), in the random and peaky regimes"""
    H, W, heads = 26, 31, 8
    for name in ('random', 'peaky'):
        qkv, table = wr.make_case(name, 1, H, W, hd * heads, heads, shift, seed=hd)
        run_case('hd %d %s shift %d' % (hd, name, shift), qkv, table, H, W, hd * heads, heads, shift)


# ------------------------------------------------------------------------------------------------ grid edges
@pytest.mark.parametrize('shift', [0, 6])
@pytest.mark.parametrize('H,W', [(12, 12), (24, 36), (25, 37), (12, 120), (120, 12), (13, 121)])
def test_grid_edges(cuda, H, W, shift):
    """one window (region 0 empty at shift 6), exact multiples of 12 (no pad), 12k + 1 (11 pad rows / columns), one
    window row or column"""
    C, heads = 64, 8
    for name in ('random', 'mask_dominance'):
        qkv, table = wr.make_case(name, 1, H, W, C, heads, shift, seed=H * W)
        run_case('%dx%d %s shift %d' % (H, W, name, shift), qkv, table, H, W, C, heads, shift)


# ------------------------------------------------------------------------------------------------ adversarial
ADVERSARIAL = ['peaky', 'mask_dominance', 'rising_max', 'hot_first_key', 'hot_last_key', 'ones_v', 'self_select',
               'offset_select']


@pytest.mark.parametrize('shift', [0, 6])
@pytest.mark.parametrize('name', ADVERSARIAL)
def test_adversarial(cuda, name, shift):
    for i, (H, W, C, heads) in enumerate([(28, 37, 256, 32), (30, 50, 32, 8), (14, 19, 16, 8)]):
        qkv, table = wr.make_case(name, 2, H, W, C, heads, shift, seed=i)
        got, _, _ = run_case('%s %dx%d C%d h%d shift %d' % (name, H, W, C, heads, shift), qkv, table, H, W, C,
                             heads, shift)
        if name == 'self_select':
            Hp, Wp = wr.padded(H, W)
            assert torch.equal(got.float(), wr.self_select_expected(2, Hp, Wp, C).cuda()), 'self_select not exact'
        if name == 'ones_v':
            assert ((got.float() - 1).abs() <= 2.0 ** -7).all(), 'ones_v: more than one bf16 ulp from 1'


def test_mask_dominance_at_level0(cuda):
    H, W, C, heads = LEVELS[0]
    qkv, table = wr.make_case('mask_dominance', 1, H, W, C, heads, 6, seed=0)
    run_case('mask_dominance level 0 shift 6', qkv, table, H, W, C, heads, 6)


# ------------------------------------------------------------------------------------------------ batched
@pytest.mark.parametrize('shift', [0, 6])
@pytest.mark.parametrize('B', [2, 3])
@pytest.mark.parametrize('H,W,C,heads', [(28, 37, 256, 32), (56, 74, 256, 16), (14, 19, 64, 16)])
def test_batched_equals_single(cuda, H, W, C, heads, B, shift):
    """blockIdx.z = image: each image of a B-image launch is bit-identical to its own B = 1 launch"""
    Hp, Wp = wr.padded(H, W)
    qkv, table = wr.make_case('peaky', B, H, W, C, heads, shift, seed=B)
    qkv, table = qkv.cuda(), table.cuda()
    batch = launch(qkv, table, Hp, Wp, C, heads, shift)
    assert torch.isfinite(batch.float()).all()
    for b in range(B):
        one = launch(qkv[b:b + 1], table, Hp, Wp, C, heads, shift)
        assert torch.equal(batch[b:b + 1], one), 'image %d of %d differs from its single launch' % (b, B)


# ------------------------------------------------------------------------------------------------ refusals
@pytest.mark.parametrize('Hp,Wp,C,heads,B', [(30, 24, 64, 8, 1), (24, 30, 64, 8, 1), (24, 24, 48, 8, 1),
                                             (24, 24, 128, 2, 1), (24, 24, 64, 8, 0)])
def test_refusals(cuda, Hp, Wp, C, heads, B):
    """a grid that is not a multiple of the window, an unsupported head dim (6, 64) or B = 0 is an error and writes
    nothing; the buffers are large enough for what a launch would address, so a missing check could not fault"""
    from patchfusion_b200.lib import PFError
    ops = _ops()
    rows = max(B, 1) * (Hp + 12) * (Wp + 12)
    qkv = torch.randn(rows, 3 * C, device=cuda).to(BF16)
    table = torch.randn(wr.NREL, heads, device=cuda)
    out = torch.full((rows, C), wr.SENTINEL, dtype=BF16, device=cuda)
    with pytest.raises(PFError):
        ops.call('pf_window_attention_batched', qkv, table, B, Hp, Wp, C, heads, 6, out, ops.stream_ptr())
    torch.cuda.synchronize()
    assert (out == wr.SENTINEL).all()


# ------------------------------------------------------------------------------------------------ batched helpers
def _f(x):
    return ctypes.c_float(x)


@pytest.mark.parametrize('H,W,C', [(28, 37, 256), (50, 61, 32)])
def test_g2l_embed_batched(cuda, H, W, C):
    """x[b] = float(feat[b, :, :C]) + ape at B = 3 with feat_ld > C: NaN in the pad columns never reaches x"""
    ops = _ops()
    g = torch.Generator(device=cuda).manual_seed(C)
    B, n, ld = 3, H * W, C + 8
    feat = torch.full((B, n, ld), float('nan'), dtype=BF16, device=cuda)
    feat[..., :C] = torch.randn(B, n, C, device=cuda, generator=g).to(BF16)
    ape = torch.randn(n, C, device=cuda, generator=g)
    x = torch.full((B * n + EXTRA, C), wr.SENTINEL, device=cuda)
    ops.call('pf_g2l_embed_batched', feat, ld, ape, B, n, C, x, ops.stream_ptr())
    torch.cuda.synchronize()
    assert torch.equal(x[:B * n].view(B, n, C), feat[..., :C].float() + ape)
    assert (x[B * n:] == wr.SENTINEL).all()


@pytest.mark.parametrize('H,W,C', [(28, 37, 256), (50, 61, 32), (13, 25, 32)])
def test_swin_norm_pad_batched(cuda, H, W, C):
    """LayerNorm into the zero-padded grids of B = 3 images: pad rows exactly 0, valid rows within the bf16 rounding
    of fp64 LayerNorm (half an ulp plus 2^-18 of |x_hat g| + |b| for the fp32 arithmetic), sentinel rows intact"""
    ops = _ops()
    g = torch.Generator(device=cuda).manual_seed(H + C)
    B = 3
    Hp, Wp = wr.padded(H, W)
    x = torch.randn(B, H * W, C, device=cuda, generator=g) * 3 + 0.7
    w = 1 + 0.3 * torch.randn(C, device=cuda, generator=g)
    b = 0.5 * torch.randn(C, device=cuda, generator=g)
    out = torch.full((B * Hp * Wp + EXTRA, C), wr.SENTINEL, dtype=BF16, device=cuda)
    ops.call('pf_swin_norm_pad_batched', x, w, b, _f(1e-5), B, H, W, Hp, Wp, C, out, ops.stream_ptr())
    torch.cuda.synchronize()
    assert (out[B * Hp * Wp:] == wr.SENTINEL).all()
    grid = out[:B * Hp * Wp].view(B, Hp, Wp, C)
    assert (grid[:, H:] == 0).all() and (grid[:, :, W:] == 0).all(), 'pad rows / columns not zeroed'
    x64 = x.double()
    xh = (x64 - x64.mean(-1, keepdim=True)) / (x64.var(-1, unbiased=False, keepdim=True) + 1e-5).sqrt()
    ref = (xh * w.double() + b.double()).view(B, H, W, C)
    got = grid[:, :H, :W].double()
    bound = 0.5 * torch.maximum(wr.bf16_ulp(ref), wr.bf16_ulp(got)) + \
        2.0 ** -18 * ((xh * w.double()).abs() + b.double().abs()).view(B, H, W, C)
    r = ((got - ref).abs() / bound).max().item()
    print('swin_norm_pad %dx%d C%d B3: %.2f of the bound' % (H, W, C, r))
    assert r <= 1.0


@pytest.mark.parametrize('H,W,C', [(28, 37, 256), (50, 61, 32)])
def test_swin_residual_crop_batched(cuda, H, W, C):
    """x[b] += y[b] cropped to H x W at B = 3: bit-identical to the torch add, NaN in y's pad never read"""
    ops = _ops()
    g = torch.Generator(device=cuda).manual_seed(W + C)
    B = 3
    Hp, Wp = wr.padded(H, W)
    x0 = torch.randn(B * H * W, C, device=cuda, generator=g)
    y = torch.full((B, Hp, Wp, C), float('nan'), device=cuda)
    y[:, :H, :W] = torch.randn(B, H, W, C, device=cuda, generator=g)
    x = torch.full((B * H * W + EXTRA, C), wr.SENTINEL, device=cuda)
    x[:B * H * W] = x0
    ops.call('pf_swin_residual_crop_batched', x, y, B, H, W, Hp, Wp, C, ops.stream_ptr())
    torch.cuda.synchronize()
    assert torch.equal(x[:B * H * W], x0 + y[:, :H, :W].reshape(B * H * W, C))
    assert (x[B * H * W:] == wr.SENTINEL).all()


# ------------------------------------------------------------------------------------------------ one Swin block
def _ln64(x, w, b):
    mu = x.mean(-1, keepdim=True)
    return (x - mu) / ((x - mu).pow(2).mean(-1, keepdim=True) + 1e-5).sqrt() * w.double() + b.double()


@pytest.mark.parametrize('B', [1, 2])
@pytest.mark.parametrize('shift', [0, 6])
@pytest.mark.parametrize('H,W,C,heads', [LEVELS[0], LEVELS[4]])
def test_swin_block_chain(cuda, H, W, C, heads, shift, B):
    """x += proj(window_attention(qkv(norm_pad(x)))) cropped, then x += fc2(gelu(fc1(LN(x)))), through the ops
    wrappers in the engine's order (pf_stage.cu g2l_run).  Each branch's update (x after minus x before) is compared
    with fp64, with bf16 rounding where the engine stores bf16 (LN outputs, qkv, attention output, hidden layer); the
    MLP branch starts from the kernels' x after the attention branch, so it carries one LN store and one hidden store
    and stays within FP64_TOL."""
    ops = _ops()
    g = torch.Generator(device=cuda).manual_seed(C + shift + B)
    Hp, Wp = wr.padded(H, W)
    rows, prow = B * H * W, B * Hp * Wp
    r = lambda *s, std=1.0: torch.randn(*s, device=cuda, generator=g) * std                       # noqa: E731
    x0 = r(rows, C, std=2.0) + 0.5
    n1w, n1b, n2w, n2b = 1 + r(C, std=0.2), r(C, std=0.2), 1 + r(C, std=0.2), r(C, std=0.2)
    wqkv, bqkv = r(3 * C, C, std=C ** -0.5), r(3 * C, std=0.5)
    wqkv[:2 * C] *= 2                                   # q, k ~ N(0, 4): logit std about 4
    table = r(wr.NREL, heads)
    wproj, bproj = r(C, C, std=C ** -0.5), r(C, std=0.2)
    w1, b1 = r(4 * C, C, std=C ** -0.5), r(4 * C, std=0.2)
    w2, b2 = r(C, 4 * C, std=(4 * C) ** -0.5), r(C, std=0.2)
    pq, pp, p1, p2 = (ops.pack_weight(a, c) for a, c in ((wqkv, bqkv), (wproj, bproj), (w1, b1), (w2, b2)))
    ones = torch.ones(C, device=cuda)

    x = x0.clone()
    npad = torch.empty(prow, C, dtype=BF16, device=cuda)
    qkv = torch.empty(prow, 3 * C, dtype=BF16, device=cuda)
    att = torch.empty(prow, C, dtype=BF16, device=cuda)
    prj = torch.empty(prow, C, device=cuda)
    hb = torch.empty(rows, C, dtype=BF16, device=cuda)
    hid = torch.empty(rows, 4 * C, dtype=BF16, device=cuda)
    ops.call('pf_swin_norm_pad_batched', x, n1w, n1b, _f(1e-5), B, H, W, Hp, Wp, C, npad, ops.stream_ptr())
    ops.gemm(pq, [npad], qkv)
    ops.call('pf_window_attention_batched', qkv, table, B, Hp, Wp, C, heads, shift, att, ops.stream_ptr())
    ops.gemm(pp, [att], prj)
    ops.call('pf_swin_residual_crop_batched', x, prj, B, H, W, Hp, Wp, C, ops.stream_ptr())
    torch.cuda.synchronize()
    x1 = x.clone()
    ops.layernorm(x, n2w, n2b, 1e-5, hb)
    ops.gemm(p1, [hb], hid, act=ops.ACT_GELU)
    ops.gemm(p2, [hid], x, gamma=ones)
    torch.cuda.synchronize()

    # attention branch in fp64
    h = wr.rb(_ln64(x0.double(), n1w, n1b)).double().view(B, H, W, C)
    h = F.pad(h, (0, 0, 0, Wp - W, 0, Hp - H)).reshape(B, Hp * Wp, C)
    q64 = wr.rb(h @ wr.rb(wqkv).double().T + bqkv.double())
    a64 = wr.rb(wr.window_attention_fp64(q64, table, Hp, Wp, C, heads, shift)).double()
    upd = (a64 @ wr.rb(wproj).double().T + bproj.double()).view(B, Hp, Wp, C)[:, :H, :W].reshape(rows, C)
    e_att = wr.rel_linf(x1.double() - x0.double(), upd)
    # MLP branch in fp64, from the kernels' x after the attention branch
    h2 = wr.rb(_ln64(x1.double(), n2w, n2b)).double()
    hid64 = wr.rb(F.gelu(h2 @ wr.rb(w1).double().T + b1.double())).double()
    upd2 = hid64 @ wr.rb(w2).double().T + b2.double()
    e_mlp = wr.rel_linf(x.double() - x1.double(), upd2)
    print('swin block %dx%d C%d h%d shift %d B%d: attention update %.2e (bound %.1e), MLP update %.2e (bound %.1e)'
          % (H, W, C, heads, shift, B, e_att, CHAIN_TOL, e_mlp, wr.FP64_TOL))
    assert e_att <= CHAIN_TOL
    assert e_mlp <= wr.FP64_TOL
