"""References and input cases shared by the Swin window-attention tests (test_gpu_window_attn.py on the GPU,
test_window_reference.py on the CPU) for `pf_window_attention` / `window_attention_kernel`.

Layout: qkv [B, Hp * Wp, 3C] (per token: q | k | v, head h at columns h * hd .. h * hd + hd of each), the
relative-position bias table [(2 * 12 - 1)^2 = 529, heads] and the output [B, Hp * Wp, C], all on the padded grid
(Hp, Wp multiples of the 12 x 12 window).  qkv holds bf16 values (what the kernel reads), kept in fp32 here.

Two references:
  window_attention_fp64      the reference's own formulation (SW:139-161, 236-256): roll by -shift, window partition,
                             softmax(q hd^-0.5 k^T + bias[relative_position_index] + mask) v, window reverse, roll back,
                             in fp64, chunked over windows.  The attention core is oracle.pf_oracle.window_attention.
  window_attention_emulated  window_attention_kernel step by step in fp32: the token / region tables it builds, q
                             pre-scaled by rsqrt(hd) log2(e), the two FMA chains over the even and odd dims, the bias and
                             the -100 mask folded into the log2 domain, the online softmax that rescales only when the
                             running maximum moves, ex2 with subnormal results flushed, the fp32 FMA chain of p v over the
                             keys and bf16(acc * (1 / l)).  ex2.approx is modelled as exact exp2 (its error is in
                             EMU_ABS).  `bug` plants one of the mistakes the GPU tests exist to catch (PLANTED_BUGS).

The case builders take a torch Generator and build on the CPU, so the GPU tests and the CPU guard use the same inputs.
"""
import math

import torch

WS = 12
NT = WS * WS
NREL = (2 * WS - 1) ** 2
LOG2E = 1.4426950408889634
SENTINEL = -1024.0               # exact in bf16; an attention output is a convex combination of V rows: never this

# ------------------------------------------------------------------------------------------------------ tolerances
# Global relative L-inf (max |got - ref| / max |ref|) of the kernel against window_attention_fp64.  The emulation
# departs from exact arithmetic by fp32 rounding and the bf16 output store; it measures at most 3.7e-3 against fp64
# over the case families of test_window_reference.py (rising_max; the half-ulp rounding of bf16 alone reaches 2^-8 =
# 3.9e-3 at an element just above a power of two near the largest).  Twice that, rounded up, is the bound.
FP64_TOL = 8e-3
# Kernel against the emulation, per element: |got - emu| <= EMU_ULPS ulp_bf16(|emu|) + EMU_ABS max |V|.  The kernel
# and the emulation perform the same fp32 operations in the same order (rsqrtf(HD) * log2e and 100 * log2e are folded
# at compile time to the fp32 products the emulation computes), except ex2.approx: its relative error of ~2^-22 per
# call on p and on the rescale factor perturbs p / l, so the fp32 outputs differ by a few 2^-22 max |V| before the
# store.  Rounding to bf16 turns that into a flip to the neighbouring bf16 value (one ulp) where the fp32 value sits
# next to a rounding boundary, or into the absolute term where the output nearly cancels (its ulp is then below the
# fp32 difference).  2^-18 leaves 16x over 2^-22.
EMU_ULPS = 1.0
EMU_ABS = 2.0 ** -18

PLANTED_BUGS = (
    'mask_log2_domain',   # s -= 100 (the mask applied without the log2(e) fold): a masked weight is e^-69, not e^-100
    'region_off_by_one',  # ry <= Hp - shift (and rx <= Wp - shift): the first row / column of region 2 joins region 1
    'bias_transposed',    # the bias read at (j - i) instead of (i - j)
    'no_rescale',         # acc is not multiplied by 2^(m_old - m_new) when the running maximum moves (l still is)
    'roll_backwards',     # source row / column (r - shift) mod Hp instead of (r + shift) mod Hp
)


# ------------------------------------------------------------------------------------------------------ helpers
def f32(x):
    return torch.tensor(x, dtype=torch.float32)


def padded(H, W):
    return math.ceil(H / WS) * WS, math.ceil(W / WS) * WS


def rb(x):
    return x.to(torch.bfloat16).float()


def bf16_ulp(x):
    x = x.double().abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(x)) - 7)


def rel_linf(got, want):
    """max |got - want| / max |want|; inf when got holds a NaN or inf"""
    got, want = got.double(), want.double()
    if not torch.isfinite(got).all():
        return math.inf
    return ((got - want).abs().max() / want.abs().max().clamp_min(1e-30)).item()


def emu_error(got, emu, qkv, C):
    """largest |got - emu| over its bound (EMU_ULPS ulp + EMU_ABS max |V|): a correct kernel gives <= 1"""
    got, emu = got.double(), emu.double()
    if not torch.isfinite(got).all():
        return math.inf
    vmax = qkv[..., 2 * C:].double().abs().max()
    bound = EMU_ULPS * bf16_ulp(emu) + EMU_ABS * vmax
    return ((got - emu).abs() / bound).max().item()


def _fma32(a, b, c):
    """fmaf: the product of two fp32 values is exact in fp64"""
    return (a.double() * b.double() + c.double()).float()


def _ex2(x):
    """ex2.approx.ftz.f32 modelled as exact: 2^x rounded to fp32 once, subnormal results flushed to zero"""
    y = torch.exp2(x.double()).float()
    return torch.where(y < 2.0 ** -126, torch.zeros_like(y), y)


def rel_index(device=None):
    from patchfusion_b200.params import relative_position_index
    return relative_position_index(WS).to(device)


# ------------------------------------------------------------------------------------------------------ fp64
def window_attention_fp64(qkv, table, Hp, Wp, C, heads, shift):
    """qkv [B, Hp * Wp, 3C] (or [Hp * Wp, 3C]), table [529, heads] -> [B, Hp * Wp, C] in fp64"""
    from oracle import pf_oracle as po
    assert shift in (0, WS // 2), 'the reference shifts by window_size // 2 only'
    squeeze = qkv.dim() == 2
    x = qkv.double().reshape(-1, Hp, Wp, 3 * C)
    B = x.shape[0]
    if shift:
        x = torch.roll(x, shifts=(-shift, -shift), dims=(1, 2))
    win = po._windows(x, WS)                                  # [B * nW, 144, 3C], image-major
    nW = (Hp // WS) * (Wp // WS)
    mask = po.shift_mask(Hp, Wp, WS, x.device).double() if shift else None
    index = rel_index(x.device)
    tab = table.double()
    out = torch.empty(B * nW, NT, C, dtype=torch.float64, device=x.device)
    chunk = max(1, 2048 // heads)
    for s in range(0, B * nW, chunk):
        e = min(s + chunk, B * nW)
        m = mask[torch.arange(s, e, device=x.device) % nW] if mask is not None else None
        out[s:e] = po.window_attention(win[s:e], tab, index, heads, m)
    o = po._unwindows(out, WS, Hp, Wp)
    if shift:
        o = torch.roll(o, shifts=(shift, shift), dims=(1, 2))
    o = o.reshape(B, Hp * Wp, C)
    return o[0] if squeeze else o


# ------------------------------------------------------------------------------------------------------ emulation
def kernel_tokens(Hp, Wp, shift, bug=None, device=None):
    """the kernel's stok / sreg tables: source token and shift region of every (window, thread), [nW, 144] each"""
    wpr = Wp // WS
    win = torch.arange((Hp // WS) * wpr)
    tid = torch.arange(NT)
    ry = (win // wpr)[:, None] * WS + (tid // WS)[None, :]
    rx = (win % wpr)[:, None] * WS + (tid % WS)[None, :]
    sgn = -1 if bug == 'roll_backwards' else 1
    oy, ox = (ry + sgn * shift) % Hp, (rx + sgn * shift) % Wp
    lt = (lambda a, b: a <= b) if bug == 'region_off_by_one' else (lambda a, b: a < b)     # noqa: E731
    hr = torch.where(ry < Hp - WS, 0, torch.where(lt(ry, Hp - shift), 1, 2))
    wr = torch.where(rx < Wp - WS, 0, torch.where(lt(rx, Wp - shift), 1, 2))
    sreg = hr * 3 + wr if shift > 0 else torch.zeros_like(hr)
    return (oy * Wp + ox).to(device), sreg.to(device)


def window_attention_emulated(qkv, table, Hp, Wp, C, heads, shift, bug=None):
    """window_attention_kernel<C / heads> in fp32 -> [B, Hp * Wp, C] (or [Hp * Wp, C]) fp32 holding bf16 values"""
    assert bug is None or bug in PLANTED_BUGS
    squeeze = qkv.dim() == 2
    dev = qkv.device
    x = qkv.float().reshape(-1, Hp * Wp, 3, heads, C // heads)
    B, hd = x.shape[0], C // heads
    stok, sreg = kernel_tokens(Hp, Wp, shift, bug, dev)
    nW = stok.shape[0]
    scale = (f32(1.0 / math.sqrt(hd)) * f32(LOG2E)).to(dev)               # rsqrtf(HD) * kLog2e
    sb = table.float() * f32(LOG2E).to(dev)                                # bias table in the log2 domain
    idx = rel_index(dev)                                                   # [i, j] -> row of the (i - j) offset
    if bug == 'bias_transposed':
        idx = idx.t()
    bias = sb[idx].permute(2, 0, 1)                                        # [heads, i, j]
    c100 = f32(100.0) if bug == 'mask_log2_domain' else f32(100.0) * f32(LOG2E)
    c100 = c100.to(dev)
    out = torch.empty(B, Hp * Wp, C, dtype=torch.float32, device=dev)
    chunk = max(1, 4096 // heads)
    for b in range(B):
        for w0 in range(0, nW, chunk):
            ws_ = slice(w0, min(w0 + chunk, nW))
            tok = x[b][stok[ws_]]                                          # [n, 144, 3, heads, hd]
            q = tok[:, :, 0].permute(0, 2, 1, 3) * scale                    # [n, heads, 144, hd]
            k = tok[:, :, 1].permute(0, 2, 1, 3)
            v = tok[:, :, 2].permute(0, 2, 1, 3)
            # the two FMA chains over even and odd dims, every (i, j) at once: [n, heads, i, j]
            s0 = torch.zeros(q.shape[0], heads, NT, NT, dtype=torch.float32, device=dev)
            s1 = torch.zeros_like(s0)
            for d in range(0, hd, 2):
                s0 = _fma32(q[..., d, None], k[..., None, :, d], s0)
                s1 = _fma32(q[..., d + 1, None], k[..., None, :, d + 1], s1)
            s = (s0 + s1) + bias
            cross = (sreg[ws_, :, None] != sreg[ws_, None, :])[:, None]      # [n, 1, i, j]
            s = torch.where(cross, s - c100, s)
            m = torch.full(s.shape[:3], -math.inf, dtype=torch.float32, device=dev)
            l = torch.zeros_like(m)
            acc = torch.zeros_like(q)
            for j in range(NT):
                sj = s[..., j]
                move = sj > m
                a = _ex2(m - sj)
                if bug != 'no_rescale':
                    acc = torch.where(move[..., None], acc * a[..., None], acc)
                l = torch.where(move, l * a, l)
                m = torch.where(move, sj, m)
                p = _ex2(sj - m)
                l = l + p
                acc = _fma32(p[..., None], v[:, :, j, None, :], acc)
            o = rb(acc * (f32(1.0).to(dev) / l)[..., None])                # [n, heads, 144, hd]
            rows = stok[ws_].reshape(-1)
            out[b, rows] = o.permute(0, 2, 1, 3).reshape(-1, C)
    return out[0] if squeeze else out


# ------------------------------------------------------------------------------------------------------ cases
def _rolled(Hp, Wp, shift):
    """for every token of the (unrolled) grid: its (iy, ix) inside its window of the rolled frame and the signs
    (sh, sw) that tell apart the shift regions a window can hold together ([Hp, Wp] each)"""
    ry = (torch.arange(Hp) - shift) % Hp
    rx = (torch.arange(Wp) - shift) % Wp
    iy, ix = (ry % WS)[:, None].expand(Hp, Wp), (rx % WS)[None, :].expand(Hp, Wp)
    # a window holds region rows {0} or {1, 2} (the last window row), and likewise for columns: 2 -> -1, else +1
    sh = torch.where(ry < Hp - WS // 2, 1.0, -1.0)[:, None].expand(Hp, Wp)
    sw = torch.where(rx < Wp - WS // 2, 1.0, -1.0)[None, :].expand(Hp, Wp)
    return iy, ix, sh, sw


def _coord_v(B, Hp, Wp, C):
    """V encoding each token's (y, x) as bf16-exact integers 1..33: channel c holds y // 16, y % 16, x // 16 or x % 16
    (+1, so no output is 0) for c % 4 = 0, 1, 2, 3"""
    y = torch.arange(Hp)[:, None].expand(Hp, Wp)
    x = torch.arange(Wp)[None, :].expand(Hp, Wp)
    digits = torch.stack([y // 16, y % 16, x // 16, x % 16], -1).float() + 1      # [Hp, Wp, 4]
    return digits[..., torch.arange(C) % 4].reshape(1, Hp * Wp, C).expand(B, -1, -1)


def _qkv(B, Hp, Wp, C, heads):
    return torch.zeros(B, Hp, Wp, 3, heads, C // heads)


def case_random(B, Hp, Wp, C, heads, shift, gen, qkv_std=1.0, table_std=1.0):
    qkv = torch.randn(B, Hp * Wp, 3 * C, generator=gen) * qkv_std
    return qkv, torch.randn(NREL, heads, generator=gen) * table_std


def case_peaky(B, Hp, Wp, C, heads, shift, gen):
    """qkv x8 and a bias table with std 5: logits with std in the tens (test_gpu_attn.py's peaky regime)"""
    return case_random(B, Hp, Wp, C, heads, shift, gen, 8.0, 5.0)


def case_mask_dominance(B, Hp, Wp, C, heads, shift, gen):
    """Every cross-region key 60-99 logits above the same-region keys of the query (uniform per query and head), set
    through q . k: with the -100 mask a cross-region key ends 1-40 below, e^-1 .. e^-40 of the weight.  Signs
    (sh, sw, sh sw) in k and -(c / 4) sqrt(hd) (sh, sw, sh sw) in q give c [regions differ] - 3c / 4; at hd = 2 only
    (sh, sw) fit, with c / 2: cross-region keys differing in one axis are then 30-50 above, in both 60-99."""
    hd = C // heads
    t = _qkv(B, Hp, Wp, C, heads)
    t[..., 2, :, :] = torch.randn(B, Hp, Wp, heads, hd, generator=gen)
    _, _, sh, sw = _rolled(Hp, Wp, WS // 2)
    sig = torch.stack([sh, sw, sh * sw], -1)[..., :3 if hd >= 4 else 2]           # [Hp, Wp, n]
    n = sig.shape[-1]
    c = 60 + 39 * torch.rand(B, Hp, Wp, heads, 1, generator=gen)
    t[..., 1, :, :n] = sig[None, :, :, None, :]
    t[..., 0, :, :n] = -(c / 4) * math.sqrt(hd) * sig[None, :, :, None, :]
    if hd > n:
        t[..., 0:2, :, n:] = 0.5 * torch.randn(B, Hp, Wp, 2, heads, hd - n, generator=gen)
    table = torch.randn(NREL, heads, generator=gen)
    return t.reshape(B, Hp * Wp, 3 * C), table


def case_rising_max(B, Hp, Wp, C, heads, shift, gen, step=0.25):
    """k[0] = j / 16 for the key at window position j and q[0] = 16 step sqrt(hd): every key's logit is `step` above
    the previous one (the bias table is N(0, 0.01)), so the running maximum moves at every same-region key"""
    hd = C // heads
    t = _qkv(B, Hp, Wp, C, heads)
    iy, ix, _, _ = _rolled(Hp, Wp, shift)
    t[..., 1, :, 0] = ((iy * WS + ix).float() / 16)[None, :, :, None]
    t[..., 0, :, 0] = 16 * step * math.sqrt(hd)
    t[..., 2, :, :] = torch.randn(B, Hp, Wp, heads, hd, generator=gen)
    return t.reshape(B, Hp * Wp, 3 * C), 0.01 * torch.randn(NREL, heads, generator=gen)


def _hot_key(B, Hp, Wp, C, heads, shift, gen, pos):
    hd = C // heads
    t = _qkv(B, Hp, Wp, C, heads)
    t[..., 0:3, :, :] = torch.randn(B, Hp, Wp, 3, heads, hd, generator=gen)
    iy, ix, _, _ = _rolled(Hp, Wp, shift)
    t[..., 1, :, 0] = ((iy * WS + ix) == pos).float()[None, :, :, None]
    t[..., 0, :, 0] = 30 * math.sqrt(hd)
    return t.reshape(B, Hp * Wp, 3 * C), torch.randn(NREL, heads, generator=gen)


def case_hot_first_key(B, Hp, Wp, C, heads, shift, gen):
    """window position 0 is 30 logits above every other key: the maximum is set by the first key and never moves"""
    return _hot_key(B, Hp, Wp, C, heads, shift, gen, 0)


def case_hot_last_key(B, Hp, Wp, C, heads, shift, gen):
    """window position 143 is 30 logits above every other key: one rescale by ~e^-30 at the last key"""
    return _hot_key(B, Hp, Wp, C, heads, shift, gen, NT - 1)


def case_ones_v(B, Hp, Wp, C, heads, shift, gen):
    """V = 1 under peaky logits: every output is 1 within a bf16 ulp"""
    qkv, table = case_random(B, Hp, Wp, C, heads, shift, gen, 4.0, 3.0)
    qkv[..., 2 * C:] = 1.0
    return qkv, table


def _select(B, Hp, Wp, C, heads, dy, dx):
    qkv = torch.zeros(B, Hp * Wp, 3 * C)
    qkv[..., 2 * C:] = _coord_v(B, Hp, Wp, C)
    table = torch.zeros(NREL, heads)
    table[(dy + WS - 1) * (2 * WS - 1) + dx + WS - 1] = 60.0
    return qkv, table


def case_self_select(B, Hp, Wp, C, heads, shift, gen):
    """q = k = 0, bias +60 at offset (0, 0): every token attends to itself (other keys weigh e^-60), so the output is
    bit-exactly the token's own V, which encodes its (y, x): roll, partition and write-back, pad tokens included"""
    return _select(B, Hp, Wp, C, heads, 0, 0)


OFFSET = (2, -3)


def case_offset_select(B, Hp, Wp, C, heads, shift, gen):
    """bias +60 at offset i - j = OFFSET only: query (iy, ix) attends to the key at (iy - 2, ix + 3) of its window
    (where that key exists and shares its region), so a transposed bias reads the opposite neighbour"""
    return _select(B, Hp, Wp, C, heads, *OFFSET)


CASES = {
    'random': case_random,
    'peaky': case_peaky,
    'mask_dominance': case_mask_dominance,
    'rising_max': case_rising_max,
    'hot_first_key': case_hot_first_key,
    'hot_last_key': case_hot_last_key,
    'ones_v': case_ones_v,
    'self_select': case_self_select,
    'offset_select': case_offset_select,
}


def make_case(name, B, H, W, C, heads, shift, seed):
    """-> qkv [B, Hp * Wp, 3C] fp32 holding bf16 values and table [529, heads] fp32, on the CPU"""
    Hp, Wp = padded(H, W)
    qkv, table = CASES[name](B, Hp, Wp, C, heads, shift, torch.Generator().manual_seed(seed))
    return rb(qkv).contiguous(), table.float().contiguous()


def self_select_expected(B, Hp, Wp, C):
    return _coord_v(B, Hp, Wp, C).contiguous()
