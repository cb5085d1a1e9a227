"""pf_attention_kernel against two references (tests/attn_ref.py), at the sequence lengths, softmax regimes, masks and
layouts where a flash-style kernel goes wrong:

  fp64       softmax(q k^T scale) v in fp64 on the bf16-rounded q / k / v: global rel-L-inf < FP64_TOL (8e-3).
  emulated   the kernel's own algorithm (128-key blocks, fp32 online softmax in the exp2 domain, bf16 P, bf16 output):
             every element within one bf16 ulp of |emulated| plus EMU_FLIP x max |V| of the head.

Every output buffer starts as a sentinel with extra rows past B * seq; the sentinel must survive there and in any
columns past D.  Further: V = 1 gives 1.0 within one bf16 ulp, layout strides and NaN padding do not change a bit,
two launches agree bit for bit, bad arguments raise PFError, and one ViT attention block (LN -> qkv GEMM with the
transposing V^T store -> attention -> proj GEMM into the fp32 residual stream) matches fp64 with and without PDL.
"""
import itertools
import os

import pytest
import torch

from attn_ref import (FP64_TOL, attention_emulated, attention_fp64, bf16_ulp, make_case, ones_v_error, per_head, rb,
                      rel_linf)

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

# The emulation rounds P and the output to bf16 where the kernel does.  What it cannot reproduce is fp32 summation
# order inside wgmma and ex2.approx against exp2; either can flip the bf16 rounding of one p.  That moves the output by
# 2^-8 (p / l) |v| <= 2^-9 |v| (only the row maximum's p, exactly 1, can exceed l / 2, and it never flips): an absolute
# error that scales with V, not with the output, and shows where P V cancels to a small output.  Measured on an H100
# (700 W) over every case here: at most 1 ulp of |emulated| plus 6.9e-4 x max |V| (logit std 30, seq 1037).
EMU_ULPS = 1.0
EMU_FLIP = 2.0 ** -10
SENTINEL = -1024.0                    # attention outputs are convex combinations of V rows: never this
EXTRA_ROWS = 8
SWEEP = [1, 2, 13, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1025, 1036, 1037]
SHAPES = [(1, 6), (2, 12), (3, 16)]   # (B, heads), cycled over the sweep


def _ops():
    from patchfusion_b200 import ops
    return ops


def _shape(seq):
    return SHAPES[SWEEP.index(seq) % len(SHAPES)] if seq in SWEEP else (2, 6)


def launch(q, k, v, scale, *, qk_extra=0, out_extra=0, seq_pad=None, vt_pad=0.0):
    """q / k / v fp32 [B, seq, heads, 64] -> the whole bf16 output buffer [B * seq + EXTRA_ROWS, heads * 64 + out_extra].
    qk columns past 2D hold NaN; V^T columns [seq, seq_pad) hold vt_pad."""
    ops = _ops()
    B, seq, heads, _ = q.shape
    D = heads * 64
    qk = torch.full((B * seq, 2 * D + qk_extra), float('nan'), dtype=torch.bfloat16, device=q.device)
    qk[:, :D] = q.reshape(B * seq, D)
    qk[:, D:2 * D] = k.reshape(B * seq, D)
    sp = ops.pad_to(seq, 8) if seq_pad is None else seq_pad
    vt = torch.full((B * D, sp), vt_pad, dtype=torch.bfloat16, device=q.device)
    vt.view(B, D, sp)[:, :, :seq] = v.reshape(B, seq, D).permute(0, 2, 1)
    out = torch.full((B * seq + EXTRA_ROWS, D + out_extra), SENTINEL, dtype=torch.bfloat16, device=q.device)
    ops.attention(qk, vt, B, seq, sp, heads, scale, out)
    return out


def valid(out, B, seq, heads):
    """[B, heads, seq, 64] fp32 view of the rows and columns the kernel owns; the sentinel must hold everywhere else"""
    D = heads * 64
    assert (out[B * seq:] == SENTINEL).all(), 'rows past B * seq were written'
    assert (out[:, D:] == SENTINEL).all(), 'columns past D were written'
    return out[:B * seq, :D].float().reshape(B, seq, heads, 64).permute(0, 2, 1, 3)


def compare(name, out, q, k, v, scale, emulated=True):
    """worst errors against both references, one image at a time (bench-sized fp64 scores do not fit at once)"""
    B, seq, heads, _ = q.shape
    got = valid(out, B, seq, heads)
    assert torch.isfinite(got).all(), '%s: non-finite output' % name
    num, den, worst, flip = 0.0, 0.0, 0.0, 0.0
    for b in range(B):
        qb, kb, vb = (per_head(t[b:b + 1])[0] for t in (q, k, v))
        ref = attention_fp64(qb, kb, vb, scale)
        num = max(num, (got[b].double() - ref).abs().max().item())
        den = max(den, ref.abs().max().item())
        if emulated:
            emu = attention_emulated(qb, kb, vb, scale)
            vmax = vb.abs().amax((-1, -2), keepdim=True)
            d = (got[b] - emu).abs()
            worst = max(worst, (d / (EMU_ULPS * bf16_ulp(emu.abs()) + EMU_FLIP * vmax)).max().item())
            flip = max(flip, ((d - bf16_ulp(emu.abs())).clamp_min(0) / vmax).max().item())
    rel = num / den
    print('%-44s fp64 rel-Linf %.2e (tol %.0e)  emulated %.2f of the bound (1 ulp + %.1e max|V|)' %
          (name, rel, FP64_TOL, worst, flip))
    assert rel < FP64_TOL, '%s: rel-Linf %.3e against fp64' % (name, rel)
    assert worst <= 1, '%s: %.2f x the bound against the emulation' % (name, worst)


def _case(name, B, seq, heads, seed=0, **kw):
    return make_case(name, B, seq, heads, 1000 * seed + seq, 'cuda', **kw)


# ------------------------------------------------------------------------------------------------- sequence sweep
@pytest.mark.parametrize('seq', SWEEP)
def test_sequence_sweep(cuda, seq):
    """1, 2, 13: one KV block, mostly masked, warpgroup 1 without valid rows; 63-65: warpgroup boundary of the query
    tile; 127-129: kv_left == 1 on the last block; 1025: last block holds 1 key; 1036 / 1037: the product's length."""
    B, heads = _shape(seq)
    q, k, v, scale = _case('random', B, seq, heads)
    compare('seq %d B%d h%d' % (seq, B, heads), launch(q, k, v, scale), q, k, v, scale)


def test_bench_size(cuda):
    q, k, v, scale = _case('random', 9, 1037, 16)
    compare('bench B9 h16 seq1037', launch(q, k, v, scale), q, k, v, scale)


@pytest.mark.parametrize('seq', [129, 1037])
@pytest.mark.parametrize('std,via', [(0.3, 'scale'), (1.0, 'scale'), (8.0, 'scale'), (30.0, 'scale'),
                                     (0.3, 'magnitude'), (8.0, 'magnitude'), (30.0, 'magnitude')])
def test_softmax_regime(cuda, seq, std, via):
    """logit std 0.3 (near flat) to 30 (one-hot), through the scale (0.0375 .. 3.75: the scale_log2 plumbing) or
    through the size of q and k at scale 0.125"""
    q, k, v, scale = _case('random', 2, seq, 6, std=std, via=via)
    compare('std %g via %s seq %d' % (std, via, seq), launch(q, k, v, scale), q, k, v, scale)


ADVERSARIAL = [('all_negative', 129), ('all_negative', 1025), ('all_negative', 1037),
               ('hot_last_key', 13), ('hot_last_key', 65), ('hot_last_key', 129), ('hot_last_key', 1037),
               ('planted_next_image', 129), ('planted_next_image', 1037),
               ('rising_max', 129), ('rising_max', 257), ('rising_max', 1037),
               ('first_block_max', 129), ('first_block_max', 1037)]


@pytest.mark.parametrize('name,seq', ADVERSARIAL)
def test_adversarial(cuda, name, seq):
    """all_negative: a leaked padded key (logit 0) outweighs every valid key; hot_last_key: one-hot on key seq - 1,
    which pins the key index of the S fragment; planted_next_image: huge-logit keys at the head of image b + 1;
    rising_max / first_block_max: the online-softmax rescale at its extremes (c flushed to 0, c = 1)."""
    B = 3 if name == 'planted_next_image' else 2
    q, k, v, scale = _case(name, B, seq, 6)
    compare('%s seq %d' % (name, seq), launch(q, k, v, scale), q, k, v, scale)


@pytest.mark.parametrize('name,seq', [('random', s) for s in SWEEP] +
                         [('all_negative', 129), ('all_negative', 1025), ('all_negative', 1037),
                          ('rising_max', 1037)])
def test_ones_v(cuda, name, seq):
    """V = 1: O and l sum the same p, so only the bf16 rounding of P separates them (< 2^-9 relative): 1.0 within one
    bf16 ulp in every valid row"""
    B, heads = _shape(seq)
    q, k, v, scale = _case(name, B, seq, heads)
    out = launch(q, k, torch.ones_like(v), scale)
    e = ones_v_error(valid(out, B, seq, heads))
    print('ones-V %s seq %d: %.1f ulp' % (name, seq, e))
    assert e <= 1


# ------------------------------------------------------------------------------------------------ layout contracts
@pytest.mark.parametrize('seq', [13, 129, 1037])
@pytest.mark.parametrize('layout', ['nan_pad', 'wide'])
def test_layout_contracts(cuda, seq, layout):
    """nan_pad: V^T columns [seq, pad_to(seq, 8)) hold NaN.  wide: qk_ld = 2D + 64 with NaN in the extra columns,
    out_ld = D + 16, seq_pad = pad_to(seq, 8) + 72 with NaN in every pad column.  Either way the output is bit-identical to the
    tight, zero-padded run: the V^T tensor map is seq wide, so TMA zero-fills the last KV tile past seq and never
    reads the pad."""
    B, heads = 2, 12
    q, k, v, scale = _case('random', B, seq, heads)
    base = valid(launch(q, k, v, scale), B, seq, heads)
    if layout == 'nan_pad':
        out = launch(q, k, v, scale, vt_pad=float('nan'))
    else:
        out = launch(q, k, v, scale, qk_extra=64, out_extra=16, seq_pad=_ops().pad_to(seq, 8) + 72, vt_pad=float('nan'))
    got = valid(out, B, seq, heads)
    assert torch.isfinite(got).all()
    assert torch.equal(got, base)


def test_determinism(cuda):
    q, k, v, scale = _case('random', 3, 1037, 16, std=8.0)
    a, b = launch(q, k, v, scale), launch(q, k, v, scale)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))


REFUSALS = [  # (what, B, seq, heads, seq_pad, qk_ld extra, out_ld extra, message)
    ('qk_ld % 8', 1, 129, 2, 136, 4, 0, 'multiples of 8'),
    ('out_ld % 8', 1, 129, 2, 136, 0, 4, 'multiples of 8'),
    ('seq_pad % 8', 1, 129, 2, 133, 0, 0, 'multiples of 8'),
    ('seq_pad < seq', 1, 129, 2, 128, 0, 0, 'seq_pad 128 < seq 129'),
    ('B = 0', 0, 129, 2, 136, 0, 0, 'empty problem'),
    ('seq = 0', 1, 0, 2, 8, 0, 0, 'empty problem'),
    ('heads = 0', 1, 129, 0, 136, 0, 0, 'empty problem'),
]


@pytest.mark.parametrize('what,B,seq,heads,seq_pad,qk_x,out_x,msg', REFUSALS, ids=[r[0] for r in REFUSALS])
def test_refusals(cuda, what, B, seq, heads, seq_pad, qk_x, out_x, msg):
    from patchfusion_b200.lib import PFError
    ops = _ops()
    D = max(heads, 1) * 64
    rows = max(B, 1) * max(seq, 1)
    qk = torch.zeros(rows, 2 * D + qk_x, dtype=torch.bfloat16, device=cuda)
    vt = torch.zeros(max(B, 1) * D, max(seq_pad, 8), dtype=torch.bfloat16, device=cuda)
    out = torch.full((rows, D + out_x), SENTINEL, dtype=torch.bfloat16, device=cuda)
    with pytest.raises(PFError, match=msg):
        ops.attention(qk, vt, B, seq, seq_pad, heads, 0.125, out)
    assert (out == SENTINEL).all()


# ------------------------------------------------------------------------------------- ViT attention block chain
def _set_options(mc, pdl):
    from patchfusion_b200 import lib
    lib.call('pf_set_option', lib.OPT_GEMM_MULTICAST, mc)
    lib.call('pf_set_option', lib.OPT_PDL, pdl)


def _env_options():
    """the values the library reads from the environment when nothing has set them (its defaults otherwise)"""
    pdl = os.environ.get('PF_OPT_PDL', os.environ.get('PF_B200_PDL', '0'))
    return int(os.environ.get('PF_OPT_GEMM_MULTICAST', '1')), int(pdl)


@pytest.mark.parametrize('B', [1, 3])
@pytest.mark.parametrize('D,heads', [(384, 6), (768, 12), (1024, 16)])
def test_vit_attention_chain(cuda, D, heads, B):
    """x += ls1 * proj(attn(LN(x))) through the ops wrappers in the order the ViT block runs them, V^T pre-filled with
    NaN and never cleared, at GEMM multicast 0 / 1 and PDL 0 / 1 with no synchronisation between launches.  The update
    x_after - x_before is compared with fp64 (bf16 rounding where the engine stores bf16: LN output, q / k / v,
    attention output); the residual itself would hide an attention error."""
    ops = _ops()
    seq = 1037
    seq_pad = ops.pad_to(seq, 8)
    g = torch.Generator(device='cuda').manual_seed(D + B)
    rows = B * seq
    x0 = torch.randn(rows, D, device=cuda, generator=g) * 2 + 0.5
    n1w = 1 + 0.2 * torch.randn(D, device=cuda, generator=g)
    n1b = 0.2 * torch.randn(D, device=cuda, generator=g)
    wqkv = torch.randn(3 * D, D, device=cuda, generator=g) / D ** 0.5
    wqkv[:2 * D] *= 2                                     # q, k ~ N(0, 4): logit std about 4
    bqkv = 0.5 * torch.randn(3 * D, device=cuda, generator=g)
    wproj = torch.randn(D, D, device=cuda, generator=g) / D ** 0.5
    bproj = 0.2 * torch.randn(D, device=cuda, generator=g)
    ls1 = 0.5 + torch.rand(D, device=cuda, generator=g)
    pq, pp = ops.pack_weight(wqkv, bqkv), ops.pack_weight(wproj, bproj)

    combos = list(itertools.product((0, 1), (0, 1)))      # (multicast, pdl)
    bufs = {}
    for c in combos:
        bufs[c] = dict(x=x0.clone(), h=torch.empty(rows, D, dtype=torch.bfloat16, device=cuda),
                       qk=torch.empty(rows, 2 * D, dtype=torch.bfloat16, device=cuda),
                       vt=torch.full((B * D, seq_pad), float('nan'), dtype=torch.bfloat16, device=cuda),
                       att=torch.empty(rows, D, dtype=torch.bfloat16, device=cuda))
    try:
        for c in combos:
            _set_options(*c)
            t = bufs[c]
            ops.layernorm(t['x'], n1w, n1b, 1e-6, t['h'])
            ops.gemm(pq, [t['h']], t['qk'], vt=t['vt'], vt_col0=2 * D, vt_seq=seq, vt_seq_pad=seq_pad)
            ops.attention(t['qk'], t['vt'], B, seq, seq_pad, heads, 0.125, t['att'])
            ops.gemm(pp, [t['att']], t['x'], gamma=ls1)
    finally:
        _set_options(*_env_options())
    torch.cuda.synchronize()

    x64 = x0.double()
    mu = x64.mean(-1, keepdim=True)
    h = rb((x64 - mu) / ((x64 - mu).pow(2).mean(-1, keepdim=True) + 1e-6).sqrt() * n1w.double() + n1b.double())
    qkv = rb(h.double() @ rb(wqkv).double().T + bqkv.double()).double()
    q, k, v = (qkv[:, i * D:(i + 1) * D].reshape(B, seq, heads, 64).permute(0, 2, 1, 3) for i in range(3))
    att = torch.cat([rb(attention_fp64(q[b], k[b], v[b], 0.125)).permute(1, 0, 2).reshape(seq, D) for b in range(B)])
    upd = ls1.double() * (att.double() @ rb(wproj).double().T + bproj.double())
    errs = {}
    for c in combos:
        d = bufs[c]['x'].double() - x64
        assert torch.isfinite(d).all(), 'multicast %d pdl %d: non-finite update' % c
        errs[c] = rel_linf(d, upd)
    print('chain D%d h%d B%d: update rel-Linf %s' % (D, heads, B, ' '.join('mc%d/pdl%d %.2e' % (c + (e,))
                                                                         for c, e in errs.items())))
    for c in combos:
        assert errs[c] < FP64_TOL, 'multicast %d pdl %d: update rel-Linf %.3e' % (c + (errs[c],))
    for mc in (0, 1):
        assert torch.equal(bufs[(mc, 1)]['x'], bufs[(mc, 0)]['x']), 'PDL changed the result at multicast %d' % mc
        assert torch.equal(bufs[(mc, 1)]['att'], bufs[(mc, 0)]['att'])
