"""References and input cases for the normed / hybrid bin-centre heads: `pf_seed_bins` (SeedBinRegressor's centres,
optionally normalised to [0, 1]) and `pf_attractor_normed` (AttractorLayer: b_new and the sorted, clipped metric
centres).  Shared by test_bin_centers_reference.py (CPU) and test_gpu_bin_centers.py.

Layouts are the kernels': S [pixels, S_ld] (the seed `_net` output), A [B, H, W, A_ld] (the even `_net` channels of
AttractorLayer, as the packer keeps them), centres [B, h, w, 64].

  *_fp64       the layer's formulas in fp64 at the fp32 parameter values the kernel receives.
  *_emulated   the kernel's fp32 algorithm: the butterfly sum, the two 32-lane Hillis-Steele scans, its operation
               order and fused multiply-adds.  `bug` plants one of PLANTED_BUGS.
"""
import math

import torch

import bins_ref as br

NBINS = br.NBINS
U = 2.0 ** -24

# ------------------------------------------------------------------------------------------------------ tolerances
# pf_seed_bins: max |got - ref64| / scale, scale = max |metric centres| (divided by max - min for the [0, 1] output).
# Each width w_k = (max - min) (S_k + 1e-3) / sum carries <= 3 roundings of its own (+1e-3, /, *) and the sum's: the
# butterfly adds 32 pair sums of positive terms in 6 levels, <= 6 u relative, and that error scales every width
# alike, so it moves an edge by <= 6 u (max - min).  The Hillis-Steele scan puts every inclusive prefix through
# <= 5 additions, the upper half one more (its offset by the lower half's total), and the edge another (+ min): all
# partial sums are positive and <= max, so <= 7 u max.  The centre's average adds one rounding of the two edges and
# the [0, 1] output two more (- min, / range) of a value <= 1.  Sum: <= (3 + 6 + 7 + 2 + 2) u = 20 u of max;
# 32 u leaves room for the fp32 range (max - min) the kernel forms itself.
SEED_TOL = 32 * U
# pf_attractor_normed, b_new: the up-sampled centre bc carries pf_attractor's chain-family coordinate error
# (bins_ref.chain_tol(h, w) relative to max |b|).  b_new = bc + agg_a dist(A_a - bc) moves with bc at the slope
# 1 - agg_a dist'(dx_a), and |dist'| <= 1, so the error is amplified by up to 1 + nA for 'sum' and 2 for 'mean' (on
# normalised centres the attractors sit within a few 1e-2 of many bins at once, where dist' is close to 1).  The
# + 1e-3 is one more rounding of each attractor point, and the sum's roundings (<= nA ulps of partial sums <= nA
# * 0.03) stay below the amplified bound.  Centres: fma(range, b, min), sorted and clipped.  Sorting two vectors
# cannot increase their largest element-wise difference, nor can the clip, so |centres - ref| <= range |b - b_ref|
# + 1 ulp of max: centers_tol, relative to max.


def attractor_tol(hw, nA, kind):
    """bound on max |b_new - ref64| / max |b_new|"""
    return br.chain_tol(*hw) * (1 + (nA if kind == 'sum' else 1))


def centers_tol(b_tol_abs, lo, hi):
    """bound on max |centres - ref64| / hi given the b_new bound b_tol_abs (absolute)"""
    return (hi - lo) * b_tol_abs / hi + 2 * U


PLANTED_BUGS = {
    'seed': (
        'no_min_pad',        # edges = cumsum(widths) without the min_depth in front
        'cumsum_shifted',    # centre k is the midpoint of edges k+1 and k+2
        'no_unit',           # the [0, 1] normalisation for the attractors skipped (hybrid2 / normed b_prev)
        'eps_dropped',       # widths from S instead of S + 1e-3
    ),
    'attractor': (
        'odd_channels',      # the odd `_net` channels read as attractor points
        'eps_dropped',       # A instead of A + 1e-3
        'sort_skipped',      # metric centres not sorted
        'clip_skipped',      # metric centres not clipped to [min, max]
    ),
}


def f32(x):
    return torch.tensor(x, dtype=torch.float32)


def _fma32(a, b, c):
    return (a.double() * b.double() + c.double()).float()


# ------------------------------------------------------------------------------------------------------ pf_seed_bins
def seed_bins_fp64(S, lo, hi, normed, to_unit):
    """S [P, >= 64] -> (centres [P, 64] fp64, scale for the error)"""
    lo, hi = float(f32(lo)), float(f32(hi))
    c = S[:, :NBINS].double()
    if normed:
        w = c + float(f32(1e-3))
        w = (hi - lo) * w / w.sum(-1, keepdim=True)
        e = lo + torch.cat([torch.zeros(c.shape[0], 1, dtype=torch.float64), torch.cumsum(w, -1)], -1)
        c = 0.5 * (e[:, :-1] + e[:, 1:])
    scale = c.abs().max().item()
    if to_unit:
        c = (c - lo) / (hi - lo)
        scale /= (hi - lo)
    return c, scale


def _scan32(v):
    """Hillis-Steele inclusive scan over 32 lanes (last dim), fp32, as __shfl_up_sync with lane >= o"""
    lane = torch.arange(32)
    for o in (1, 2, 4, 8, 16):
        t = torch.cat([torch.zeros(*v.shape[:-1], o), v[..., :-o]], -1)
        v = torch.where(lane >= o, v + t, v)
    return v


def seed_bins_emulated(S, lo, hi, flags, bug=None):
    """seed_bins_kernel in fp32 -> [P, 64]"""
    assert bug is None or bug in PLANTED_BUGS['seed']
    lo, hi = f32(lo), f32(hi)
    rng = hi - lo
    c = S[:, :NBINS].float()
    if flags & 1:
        w = c if bug == 'eps_dropped' else c + f32(1e-3)
        s = w[:, :32] + w[:, 32:]
        lane = torch.arange(32)
        for o in (16, 8, 4, 2, 1):
            s = s + s[:, lane ^ o]
        w = rng * (w / s[:, :1])
        inc = [_scan32(w[:, :32]), _scan32(w[:, 32:])]
        exc = [torch.cat([torch.zeros(c.shape[0], 1), x[:, :-1]], -1) for x in inc]
        half = inc[0][:, 31:32]
        exc[1] = torch.cat([half, exc[1][:, 1:] + half], -1)
        inc[1] = inc[1] + half
        inc, exc = torch.cat(inc, -1), torch.cat(exc, -1)
        base = f32(0.0) if bug == 'no_min_pad' else lo
        if bug == 'cumsum_shifted':
            exc, inc = inc, torch.cat([inc[:, 1:], inc[:, -1:] + w[:, -1:]], -1)
        c = f32(0.5) * ((base + exc) + (base + inc))
    if flags & 2 and bug != 'no_unit':
        c = (c - lo) / rng
    return c


def seed_error(got, ref, scale):
    got = got.double()
    if not torch.isfinite(got).all():
        return math.inf
    return ((got - ref).abs().max() / max(scale, 1e-30)).item()


def seed_case(P, gen, ld=64):
    """S [P, ld] seed `_net` outputs (NaN in the columns >= 64), each pixel one of: ReLU-like (many exact zeros), all
    zero, one dominant bin, tiny values where the 1e-3 dominates, softplus-like."""
    def part(k, n):
        r = torch.randn(n, NBINS, generator=gen)
        if k == 'relu':
            return r.clamp_min(0)
        if k == 'zero':
            return torch.zeros(n, NBINS)
        if k == 'dominant':
            x = r.clamp_min(0) * 1e-2
            x[torch.arange(n), torch.randint(0, NBINS, (n,), generator=gen)] = 1e4
            return x
        if k == 'tiny':
            return r.abs() * 1e-4
        if k == 'softplus':
            return torch.nn.functional.softplus(3 * r) * 20
        raise ValueError(k)
    kinds = ('relu', 'zero', 'dominant', 'tiny', 'softplus')
    pick = torch.randint(0, len(kinds), (P,), generator=gen)
    S = torch.stack([part(k, P) for k in kinds])[pick, torch.arange(P)]
    out = torch.full((P, ld), float('nan'))
    out[:, :NBINS] = S
    return out


# ------------------------------------------------------------------------------------------------ pf_attractor_normed
def attractor_normed_fp64(A2, nA, b_prev, lo, hi, kind, typ):
    """A2 [B, H, W, >= 2 nA] (all `_net` channels, ReLU'd), b_prev [B, h, w, 64] -> (b_new, centres, delta) fp64"""
    lo, hi = float(f32(lo)), float(f32(hi))
    A = A2[..., 0:2 * nA:2].double() + float(f32(1e-3))
    b, d = br.attractor_fp64(A, nA, b_prev, kind, typ)
    c = torch.sort((hi - lo) * b + lo, -1).values.clamp(lo, hi)
    return b, c, d


def attractor_normed_emulated(A2, nA, b_prev, flags, lo, hi, bug=None):
    """attractor_normed_kernel in fp32 -> (b_new, centres)"""
    assert bug is None or bug in PLANTED_BUGS['attractor']
    A = A2[..., 1:2 * nA:2] if bug == 'odd_channels' else A2[..., 0:2 * nA:2]
    A = A.float() if bug == 'eps_dropped' else A.float() + f32(1e-3)
    b = br.attractor_emulated(A.contiguous(), nA, b_prev, flags)
    lo, hi = f32(lo), f32(hi)
    c = _fma32(hi - lo, b, lo)
    if bug != 'sort_skipped':
        c = torch.sort(c, -1).values
    if bug != 'clip_skipped':
        c = torch.minimum(torch.maximum(c, lo), hi)
    return b, c


ORDERS = ('sorted', 'reversed', 'interleaved', 'ties', 'equal', 'outside')


def unit_bins(shape, gen, order):
    """[..., 64] normalised bin centres in one of ORDERS: 'outside' spans [-0.2, 1.2] (the clip decides), the others
    [0, 1] sorted, reversed, alternating low / high, on four tied levels, or all equal"""
    b = torch.sort(torch.rand(*shape, NBINS, generator=gen), -1).values
    if order == 'reversed':
        b = b.flip(-1)
    elif order == 'interleaved':
        b = torch.cat([b[..., :32, None], b[..., 32:, None].flip(-2)], -1).reshape(*shape, NBINS)
    elif order == 'ties':
        b = torch.floor(torch.rand(*shape, NBINS, generator=gen) * 4) / 3
    elif order == 'equal':
        b = torch.rand(*shape, 1, generator=gen).expand(*shape, NBINS).contiguous()
    elif order == 'outside':
        b = torch.rand(*shape, NBINS, generator=gen) * 1.4 - 0.2
    return b


def attractor_normed_case(B, hw, HW, nA, gen, order='sorted', sigma=0.06, A_ld=32):
    """A2 [B, H, W, 2 A_ld]: even channels near a random up-sampled bin (ReLU'd, so some are exact zeros), odd channels
    far away (a kernel given the odd ones moves b visibly); A [B, H, W, A_ld] the even ones as the packer keeps them,
    NaN in the columns >= nA; b_prev [B, h, w, 64]."""
    (h, w), (H, W) = hw, HW
    b_prev = unit_bins((B, h, w), gen, order)
    bu = torch.nn.functional.interpolate(b_prev.double().permute(0, 3, 1, 2), size=(H, W), mode='bilinear',
                                         align_corners=True).permute(0, 2, 3, 1)
    k = torch.randint(0, NBINS, (B, H, W, nA), generator=gen)
    a = (torch.gather(bu, -1, k) + sigma * torch.randn(B, H, W, nA, generator=gen, dtype=torch.float64)).clamp_min(0)
    A2 = torch.full((B, H, W, 2 * A_ld), float('nan'))
    A2[..., 0:2 * nA:2] = a.float()
    A2[..., 1:2 * nA:2] = (2.0 + torch.rand(B, H, W, nA, generator=gen)).float()
    A = torch.full((B, H, W, A_ld), float('nan'))
    A[..., :nA] = a.float()
    return A2, A, b_prev.float()


def attractor_errors(b, c, b_ref, c_ref, lo, hi, hw, nA, kind):
    """(b error / its bound, centres error / its bound); a correct kernel gives <= 1 for both"""
    if not (torch.isfinite(b).all() and torch.isfinite(c).all()):
        return math.inf, math.inf
    b_tol = attractor_tol(hw, nA, kind)
    bmax = b_ref.abs().max().item()
    eb = (b.double() - b_ref).abs().max().item() / (b_tol * bmax)
    ec = (c.double() - c_ref).abs().max().item() / float(f32(hi)) / centers_tol(b_tol * bmax, lo, hi)
    return eb, ec
