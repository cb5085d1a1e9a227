"""References and input cases shared by the metric-bins tail tests (test_gpu_bins_tail.py on the GPU,
test_bins_reference.py on the CPU) for `pf_attractor`, `pf_logbinom_depth` and `pf_add_upsampled`.

All tensors are in the kernels' layouts: A [B, H, W, A_ld], bin centres [B, h, w, 64], pt [B, H, W, pt_ld],
embeddings [B, H, W, C] (bf16).  Up-sampling is bilinear with align_corners=True throughout.

Two kinds of reference:
  *_fp64       the operation in fp64 (F.interpolate on fp64, the reference's formulas), parameters taken at the fp32
               values the kernel receives.
  *_emulated   the kernel's fp32 algorithm step by step: its coordinate arithmetic (fp32 scale, truncation, clamped
               `hi` index) with reads from the flat buffer the kernel indexes, its operation order, its reductions.
               `bug` plants one of the mistakes the GPU tests exist to catch (PLANTED_BUGS).

Two input families for the attractor:
  exact   dyadic resize ratios, bins on a 2^-8 grid and A on a 2^-12 grid: the fp32 up-sample and dx = A - b are exact,
          so after the one rounding of the output store the only error left is that of the attractor function and its
          sum, and the bound is relative to the largest shift max |delta|.
  chain   the model's resize ratios and real-valued bins in [1e-3, 80]: the bound is relative to max |b|.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

NBINS = 64
MIN_TEMP, MAX_TEMP = 0.0212, 50.0        # the shipped configs (configs.py)
SENTINEL = -1024.0          # exact in fp32 and bf16

# The head's resize chain (level, (h, w) -> (H, W), nA in the configs) and its exact-family twin at dyadic ratios.
CHAIN = [((14, 19), (28, 37), 16), ((28, 37), (56, 74), 8), ((56, 74), (112, 148), 4), ((112, 148), (224, 296), 1)]
EXACT_CHAIN = [((15, 19), (29, 37), 16), ((29, 37), (57, 73), 8), ((57, 73), (113, 145), 4), ((113, 145), (225, 289), 1)]
ATTRACTOR_FLAGS = {0: ('sum', 'inv'), 1: ('mean', 'inv'), 2: ('sum', 'exp'), 3: ('mean', 'exp')}

# ------------------------------------------------------------------------------------------------------ tolerances
# pf_attractor, exact family: max(0, |got - ref| - 0.5 ulp32(ref)) / max |delta_fp64|.  With dx exact, what is left is
# the fp32 evaluation of dist(dx) (dx * dx, 300 *, 1 +, one IEEE division or __expf: a few ulps of each term), the sum
# of up to 16 terms (16 ulps of the largest partial sum) and the division by nA (exact: nA is a power of two).  Terms
# are at most 0.03 and sums at most 16 * 0.03, so this is <= ~20 * 2^-24 * 0.5 / max|delta|: about 1e-6 at the
# smallest max |delta| the cases reach (2e-3); 1e-5 leaves a factor of 10.
ATT_EXACT_TOL = 1e-5
# pf_attractor, chain family: max |got - ref| / max |b|.  The fp32 source coordinate differs from the exact one by up to
# about 2^-24 * (h - 1) pixels per axis (the rounded scale (h-1)/(H-1), then its product with the output index), which
# moves b by that times its step between neighbouring pixels (a fraction of max |b| for sorted random bins); the blend
# adds a few ulps of |b|.  dx = A - b inherits the error of b and dist has slope <= 1 near dx = 0, so the shift adds at
# most as much again per attractor close to a bin.  2^-24 * (h + w) grows with the source size as that coordinate error
# does; the emulation stays 5x or more below it at every level of the chain (3.1e-6 against 1.55e-5 at 112 x 148).


def chain_tol(h, w):
    return 2.0 ** -24 * (h + w)


# pf_logbinom_depth: relative L-inf against logbinom_depth_fp64 <= max(4 x the error of the reference's own fp32
# formula (oracle.pf_oracle.log_binomial_depth) on the same inputs, LOGBINOM_FLOOR).  The fp32 formula errs by the
# rounding of y (|y| up to 63 ln 63 = 261, ulp 3e-5) divided by t: up to 1.4e-3 in an exponent at t = min_temp, so the
# bound scales with the regime.  The kernel computes the same exponent through fmaf(logc, 1/t, ...) and __logf,
# __expf, __fdividef: each adds a few ulps of |y / t| and of the weights, so its error tracks the formula's within a
# small factor.  In the flat regime the formula's error is a few fp32 ulps of the depth; the floor, 32 ulps (2^-19),
# covers the kernel's intrinsics and its different summation order there.
LOGBINOM_FLOOR = 2.0 ** -19

# pf_add_upsampled: |got - bf16(ref64)| <= 1 bf16 ulp of |ref64| + ADD_FP32_SLACK * (|a| + up(|prev|))
# + chain_tol(h, w) * max |prev|.  The kernel evaluates a + sum w q in fp32 (4 products with 24-bit weights, 4 adds:
# under 8 ulps of the operand magnitudes) at fp32 coordinates (the chain-family coordinate error above) and rounds once;
# only where a and up(prev) nearly cancel do those fp32 errors exceed a bf16 ulp of the small result.
ADD_FP32_SLACK = 2.0 ** -21

PLANTED_BUGS = {
    'attractor': (
        'align_corners_false',  # half-pixel source coordinates (src = (dst + 0.5) * h / H - 0.5)
        'mean_sum_swapped',     # kind_mean read inverted
        'inv_exp_swapped',      # type_exp read inverted
        'image0_only',          # every image reads image 0's b_prev
        'hi_unclamped',         # hi = lo + 1 also at the last row / column (reads past the row / the buffer)
        'no_mean_divide',       # s /= nA dropped
    ),
    'logbinom': (
        'p_clamp_dropped',      # pr = min(pr, 1) only: p below 1e-4 is not raised to 1e-4
        'q_clamp_dropped',      # om = min(1 - pr, 1) only: 1 - p below 1e-4 (down to 0) is used as is
        'temp_multiplied',      # y * t instead of y / t
        'bins_reversed',        # weight of bin k paired with bin centre 63 - k
        'no_butterfly',         # max and sums over one lane's 8 bins only
        'butterfly_two_steps',  # the 8-lane butterflies stop after xor 4 and xor 2
        'bins_scale',           # bin centres sampled at scale h / H instead of (h - 1) / (H - 1)
    ),
    'add_upsampled': (
        'align_corners_false',
    ),
}


# ------------------------------------------------------------------------------------------------------ helpers
def f32(x):
    return torch.tensor(x, dtype=torch.float32)


def ulp32(x):
    """spacing of fp32 values at |x| (normal range)"""
    x = x.double().abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(x)) - 23)


def bf16_ulp(x):
    x = x.double().abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(x)) - 7)


def ac_scale(n_in, n_out):
    """the host's fp32 align_corners scale (pf_elem.cu ac_scale)"""
    return (f32(n_in - 1) / f32(n_out - 1)) if n_out > 1 else f32(0.0)


def ac_coord(n_out, n_in, bug=None, scale=None):
    """pf_elem.cu ac_coord_s for every output index: (lo, hi, frac) with frac in fp32"""
    dst = torch.arange(n_out, dtype=torch.float32)
    if bug == 'align_corners_false':
        src = ((dst + 0.5) * f32(n_in / n_out) - 0.5).clamp_min(0)
    else:
        src = (ac_scale(n_in, n_out) if scale is None else f32(scale)) * dst
    lo = src.long().clamp(max=n_in - 1)
    hi = lo + 1 if bug == 'hi_unclamped' else torch.where(lo < n_in - 1, lo + 1, lo)
    return lo, hi, src - lo.float()


def _flat_with_tail(x):
    """the buffer a kernel indexes, followed by one image row of NaN (what a read past the end would meet)"""
    B, h, w, C = x.shape
    return torch.cat([x.reshape(-1), torch.full(((w + 1) * C,), float('nan'), dtype=x.dtype)])


def _bilinear_taps(src, B, H, W, bug=None, scale=None):
    """the four tap row offsets (into the flat buffer, in elements / C) and fy, fx for every output pixel"""
    _, h, w, _ = src.shape
    y0, y1, fy = ac_coord(H, h, bug, None if scale is None else scale[0])
    x0, x1, fx = ac_coord(W, w, bug, None if scale is None else scale[1])
    img = torch.zeros(B, dtype=torch.long) if bug == 'image0_only' else torch.arange(B)
    base = (img * h * w).view(B, 1, 1)
    r = lambda yy, xx: base + (yy * w).view(1, H, 1) + xx.view(1, 1, W)          # noqa: E731
    return (r(y0, x0), r(y0, x1), r(y1, x0), r(y1, x1)), fy.view(1, H, 1, 1), fx.view(1, 1, W, 1)


def _gather(flat, rows, C):
    idx = rows.unsqueeze(-1) * C + torch.arange(C)
    return flat[idx]


def rel_linf(got, want):
    """max |got - want| / max |want|; inf when got holds a NaN or inf"""
    got, want = got.double(), want.double()
    if not torch.isfinite(got).all():
        return math.inf
    return ((got - want).abs().max() / want.abs().max().clamp_min(1e-30)).item()


# ------------------------------------------------------------------------------------------------------ pf_attractor
def attractor_fp64(A, nA, b_prev, kind, typ):
    """A [B, H, W, >= nA], b_prev [B, h, w, 64] -> (b [B, H, W, 64], delta [B, H, W, 64]) in fp64"""
    H, W = A.shape[1:3]
    b = F.interpolate(b_prev.double().permute(0, 3, 1, 2), size=(H, W), mode='bilinear', align_corners=True)
    b = b.permute(0, 2, 3, 1)
    dx = A[..., :nA].double().unsqueeze(-1) - b.unsqueeze(-2)                   # [B, H, W, nA, 64]
    d = torch.exp(-300.0 * dx * dx) * dx if typ == 'exp' else dx / (1 + 300.0 * dx * dx)
    d = d.mean(-2) if kind == 'mean' else d.sum(-2)
    return b + d, d


def attractor_emulated(A, nA, b_prev, flags, bug=None):
    """attractor_kernel in fp32: bilinear blend as written, attractors added one by one, then / nA for the mean"""
    assert bug is None or bug in PLANTED_BUGS['attractor']
    B, H, W = A.shape[:3]
    kind_mean, type_exp = bool(flags & 1), bool(flags & 2)
    if bug == 'mean_sum_swapped':
        kind_mean = not kind_mean
    if bug == 'inv_exp_swapped':
        type_exp = not type_exp
    (r00, r01, r10, r11), fy, fx = _bilinear_taps(b_prev, B, H, W, bug)
    flat = _flat_with_tail(b_prev.float())
    q = [_gather(flat, r, NBINS) for r in (r00, r01, r10, r11)]
    one = f32(1.0)
    bc = (one - fy) * ((one - fx) * q[0] + fx * q[1]) + fy * ((one - fx) * q[2] + fx * q[3])
    s = torch.zeros_like(bc)
    for a in range(nA):
        dx = A[..., a:a + 1].float() - bc
        s = s + (torch.exp(f32(-300.0) * dx * dx) * dx if type_exp else dx / (one + f32(300.0) * dx * dx))
    if kind_mean and bug != 'no_mean_divide':
        s = s / f32(nA)
    return bc + s


def attractor_exact_error(got, ref, delta):
    """exact family: the error beyond the one rounding of the store, relative to max |delta|"""
    got, ref = got.double(), ref.double()
    if not torch.isfinite(got).all():
        return math.inf
    ex = ((got - ref).abs() - 0.5 * torch.maximum(ulp32(ref), ulp32(got))).clamp_min(0)
    # a shift of 0 everywhere (exponential attractors far from every bin) leaves b rounded once: any excess fails
    return (ex.max() / delta.abs().max().clamp_min(1e-30)).item()


def sorted_bins(shape, gen, lo=1e-3, hi=80.0, grid=None):
    """[..., 64] sorted per pixel, spanning [lo, hi] (the first and last bin pinned there); on a grid of 2^-grid"""
    b = lo + torch.rand(*shape, NBINS, generator=gen) * (hi - lo)
    b[..., 0], b[..., -1] = lo, hi
    b = torch.sort(b, dim=-1).values
    if grid is not None:
        b = torch.round(b * 2 ** grid) / 2 ** grid
    return b


def attractor_case(B, hw, HW, nA, gen, family='chain', sigma=0.06, far=False, A_ld=32):
    """A [B, H, W, A_ld] (NaN in the columns >= nA) and b_prev [B, h, w, 64].  Each attractor is the up-sampled
    centre of a random bin of its pixel plus N(0, sigma), or (far) 100-120 m, beyond every bin."""
    (h, w), (H, W) = hw, HW
    if family == 'exact':
        from exact_ref import dyadic_ratio
        dyadic_ratio(h, H), dyadic_ratio(w, W)
    b_prev = sorted_bins((B, h, w), gen, grid=8 if family == 'exact' else None)
    bu = F.interpolate(b_prev.double().permute(0, 3, 1, 2), size=(H, W), mode='bilinear', align_corners=True)
    bu = bu.permute(0, 2, 3, 1)
    if far:
        a = 100.0 + 20.0 * torch.rand(B, H, W, nA, generator=gen, dtype=torch.float64)
    else:
        k = torch.randint(0, NBINS, (B, H, W, nA), generator=gen)
        a = torch.gather(bu, -1, k) + sigma * torch.randn(B, H, W, nA, generator=gen, dtype=torch.float64)
    if family == 'exact':
        a = torch.round(a * 2 ** 12) / 2 ** 12
    A = torch.full((B, H, W, A_ld), float('nan'))
    A[..., :nA] = a.float()
    return A, b_prev.float()


# ------------------------------------------------------------------------------------------------ pf_logbinom_depth
def logc_fp32():
    """the Stirling log C(63, k) of logbinom_depth_kernel, per bin, in fp32"""
    n_ = f32(NBINS - 1) + f32(1e-7)
    k_ = torch.arange(NBINS, dtype=torch.float32) + f32(1e-7)
    return n_ * torch.log(n_) - k_ * torch.log(k_) - (n_ - k_) * torch.log(n_ - k_ + f32(1e-7))


def _temps(min_t, max_t):
    """the fp32 values the kernel receives, as Python floats"""
    return float(np.float32(min_t)), float(np.float32(max_t))


def logbinom_depth_fp64(pt, bc, H, W, min_t=MIN_TEMP, max_t=MAX_TEMP):
    """pt [B, H, W, >= 4], bc [B, h, w, 64] -> depth [B, H, W] in fp64 (ConditionalLogBinomial + expectation)"""
    min_t, max_t = _temps(min_t, max_t)
    q = pt[..., :4].double()
    p = (q[..., 0] + 1e-4) / (q[..., 0] + q[..., 1] + 2e-4)
    t = (q[..., 2] + 1e-4) / (q[..., 2] + q[..., 3] + 2e-4)
    t = ((max_t - min_t) * t + min_t).unsqueeze(-1)
    k = torch.arange(NBINS, dtype=torch.float64)
    n_, k_ = (NBINS - 1) + 1e-7, k + 1e-7
    logc = n_ * math.log(n_) - k_ * torch.log(k_) - (n_ - k_) * torch.log(n_ - k_ + 1e-7)
    lq = torch.log(torch.clamp(1 - p, 1e-4, 1)).unsqueeze(-1)
    lp = torch.log(torch.clamp(p, 1e-4, 1)).unsqueeze(-1)
    y = logc + k * lp + (NBINS - 1 - k) * lq
    prob = torch.softmax(y / t, dim=-1)
    cu = F.interpolate(bc.double().permute(0, 3, 1, 2), size=(H, W), mode='bilinear', align_corners=True)
    return (prob * cu.permute(0, 2, 3, 1)).sum(-1)


def logbinom_depth_oracle32(pt, bc, H, W, min_t=MIN_TEMP, max_t=MAX_TEMP):
    """the reference's own fp32 formula (oracle.pf_oracle.log_binomial_depth) on the same inputs -> [B, H, W]"""
    from oracle import pf_oracle as po
    min_t, max_t = _temps(min_t, max_t)
    d = po.log_binomial_depth(pt[..., :4].float().permute(0, 3, 1, 2), bc.float().permute(0, 3, 1, 2), min_t, max_t)
    return d[:, 0]


def _fma32(a, b, c):
    """fmaf: the product of two fp32 values is exact in fp64"""
    return (a.double() * b.double() + c.double()).float()


def logbinom_depth_emulated(pt, bc, H, W, min_t=MIN_TEMP, max_t=MAX_TEMP, bug=None):
    """logbinom_depth_kernel in fp32: logc per bin, inv_t, the fmaf nesting, the max-subtracted exp, the per-lane sums
    over 8 bins and the xor 4 / 2 / 1 butterflies of the 8-lane group -> depth [B, H, W]"""
    assert bug is None or bug in PLANTED_BUGS['logbinom']
    B = pt.shape[0]
    min_t, max_t = f32(min_t), f32(max_t)
    q = pt[..., :4].float().reshape(-1, 4, 1)
    p0, p1, t0, t1 = (q[:, i] + f32(1e-4) for i in range(4))
    pr, tt = p0 / (p0 + p1), t0 / (t0 + t1)
    tt = (max_t - min_t) * tt + min_t
    om = (f32(1.0) - pr).clamp_max(1.0) if bug == 'q_clamp_dropped' else (f32(1.0) - pr).clamp(1e-4, 1.0)
    pr = pr.clamp_max(1.0) if bug == 'p_clamp_dropped' else pr.clamp(1e-4, 1.0)
    inv_t = tt if bug == 'temp_multiplied' else f32(1.0) / tt
    lp, lq = torch.log(pr) * inv_t, torch.log(om) * inv_t
    kf = torch.arange(NBINS, dtype=torch.float32)
    km1 = f32(NBINS - 1)
    y = _fma32(logc_fp32().expand(q.shape[0], NBINS), inv_t.expand(-1, NBINS), _fma32(kf, lp, (km1 - kf) * lq))
    # bin centres, up-sampled as the kernel does
    bh, bw = bc.shape[1:3]
    scale = (bh / H, bw / W) if bug == 'bins_scale' else None
    (r00, r01, r10, r11), fy, fx = _bilinear_taps(bc, B, H, W, scale=scale)
    flat = _flat_with_tail(bc.float())
    one = f32(1.0)
    w00, w01, w10, w11 = (one - fy) * (one - fx), (one - fy) * fx, fy * (one - fx), fy * fx
    g = [_gather(flat, r, NBINS) for r in (r00, r01, r10, r11)]
    cv = (w00 * g[0] + w01 * g[1] + w10 * g[2] + w11 * g[3]).reshape(-1, NBINS)
    if bug == 'bins_reversed':
        cv = cv.flip(-1)
    # lane j owns bins 8j .. 8j+7; lane 0 of the group writes
    lanes = y.view(-1, 8, 8)
    steps = {'no_butterfly': 0, 'butterfly_two_steps': 2}.get(bug, 3)

    def butterfly(v, op):                           # v [P, 8 lanes] -> lane 0's value after `steps` xor steps
        for o in (4, 2, 1)[:steps]:
            v = op(v, v[:, torch.arange(8) ^ o])
        return v[:, 0]

    mx = butterfly(lanes.amax(-1), torch.maximum)
    e = torch.exp(lanes - mx.view(-1, 1, 1))
    cvl = cv.view(-1, 8, 8)
    den = torch.zeros(e.shape[:2])
    num = torch.zeros(e.shape[:2])
    for i in range(8):
        den = den + e[..., i]
        num = _fma32(e[..., i], cvl[..., i], num)
    # lanes other than 0 only feed lane 0 through the butterfly; with fewer steps lane 0 sees fewer lanes
    den, num = butterfly(den, torch.add), butterfly(num, torch.add)
    return (num / den).view(B, H, W)


REGIMES = ('mid', 'sharp', 'flat', 'p_low', 'q_low', 'mix')


def _pt_regime(name, n, gen):
    """[n, 4] softplus outputs (p0, p1, t0, t1) for one regime"""
    sp = lambda: F.softplus(torch.randn(n, generator=gen))                        # noqa: E731
    big = lambda: 1e3 * (1 + torch.rand(n, generator=gen))                        # noqa: E731
    zero = torch.zeros(n)
    if name == 'mid':          # today's inputs: t around 25
        cols = (sp(), sp(), sp(), sp())
    elif name == 'sharp':      # t -> min_temp (t0 = 0, t1 ~ 1e3: t = min_temp + ~5e-6)
        cols = (sp(), sp(), zero, big())
    elif name == 'flat':       # t -> max_temp
        cols = (sp(), sp(), big(), zero)
    elif name == 'p_low':      # p ~ 1e-7 .. 1e-8, below the 1e-4 clamp
        cols = (zero, 10 * big(), sp(), sp())
    elif name == 'q_low':      # 1 - p ~ 1e-7 .. 1e-8 (0 in fp32), below the 1e-4 clamp
        cols = (10 * big(), zero, sp(), sp())
    else:
        raise ValueError(name)
    return torch.stack(cols, -1)


def logbinom_case(B, bhw, HW, regime, gen, pt_ld=8):
    """pt [B, H, W, pt_ld] (NaN in the columns >= 4) and bin centres [B, h, w, 64] sorted and spanning [1e-3, 80]"""
    (bh, bw), (H, W) = bhw, HW
    n = B * H * W
    if regime == 'mix':        # a per-pixel mix of every regime
        pick = torch.randint(0, 5, (n,), generator=gen)
        parts = torch.stack([_pt_regime(r, n, gen) for r in REGIMES[:5]])       # [5, n, 4]
        q = parts[pick, torch.arange(n)]
    else:
        q = _pt_regime(regime, n, gen)
    pt = torch.full((B, H, W, pt_ld), float('nan'))
    pt[..., :4] = q.view(B, H, W, 4)
    return pt, sorted_bins((B, bh, bw), gen)


def logbinom_tol(oracle_err):
    return max(4 * oracle_err, LOGBINOM_FLOOR)


# ---------------------------------------------------------------------------------------------- pf_add_upsampled
def add_upsampled_fp64(a, prev):
    """a [B, H, W, C], prev [B, h, w, C] (bf16) -> a + up(prev) in fp64, and the same with |.| (for the slack)"""
    H, W = a.shape[1:3]
    u = lambda x: F.interpolate(x.double().permute(0, 3, 1, 2), size=(H, W), mode='bilinear',   # noqa: E731
                                align_corners=True).permute(0, 2, 3, 1)
    return a.double() + u(prev), a.double().abs() + u(prev.abs())


def add_upsampled_emulated(a, prev, bug=None):
    """add_upsampled_kernel in fp32, rounded to bf16 once"""
    assert bug is None or bug in PLANTED_BUGS['add_upsampled']
    B, H, W, C = a.shape
    (r00, r01, r10, r11), fy, fx = _bilinear_taps(prev, B, H, W, bug)
    flat = _flat_with_tail(prev.float())
    one = f32(1.0)
    w00, w01, w10, w11 = (one - fy) * (one - fx), (one - fy) * fx, fy * (one - fx), fy * fx
    g = [_gather(flat, r, C) for r in (r00, r01, r10, r11)]
    return (a.float() + w00 * g[0] + w01 * g[1] + w10 * g[2] + w11 * g[3]).to(torch.bfloat16)


def add_upsampled_error(got, a, prev):
    """largest |got - bf16(ref)| over its bound (1 bf16 ulp of |ref| + the fp32 slack): a correct kernel gives <= 1"""
    ref, mag = add_upsampled_fp64(a, prev)
    g = got.double()
    if not torch.isfinite(g).all():
        return math.inf
    bound = bf16_ulp(ref) + ADD_FP32_SLACK * mag + chain_tol(*prev.shape[1:3]) * prev.double().abs().max()
    return ((g - ref.to(torch.bfloat16).double()).abs() / bound).max().item()


def add_upsampled_case(B, hw, HW, C, gen):
    (h, w), (H, W) = hw, HW
    a = torch.randn(B, H, W, C, generator=gen).to(torch.bfloat16)
    prev = torch.randn(B, h, w, C, generator=gen).to(torch.bfloat16)
    return a, prev
