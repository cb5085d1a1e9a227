"""Bit-exact probes for the tensor-core GEMM and conv kernels (`pf_gemm_kernel`, `pf_conv3_halo_kernel`).

With small-integer operands every product is exact, and every partial sum below 2^24 is exact in fp32 whatever the
summation order or tensor-core grouping.  The only rounding left is the final round-to-nearest-even store to the output
dtype, which torch reproduces bit for bit.  So a kernel output must EQUAL `reference.to(out dtype)`, and any indexing,
masking or pipelining error (one product term lost, doubled or read from the wrong pixel) shows up as a mismatch whose
coordinates name the m-tile, n-tile and pixel tile it sits in (`mismatch_report`).

Operands:
- activations: integers in [-amax, amax] (default 2); residuals the same;
- weights: integers in {-1, 0, 1}, each kept with probability `density` (sparse weights keep outputs small, so that a
  +-1 error stays visible after the bf16 store: bf16 holds every integer up to 256);
- biases: integers in [-8, 8]; `gamma` and the BatchNorm-fold `scale`: powers of two.

Each generator returns `(tensor, bound)`: the largest |value| (activations, biases), or the largest L1 norm of one
output's weights.  `psum_bound` combines them into a bound on every partial sum, which `check_bound` keeps <= 2^20, a wide
margin below 2^24.  The references are F.linear / F.conv2d / F.conv_transpose2d / F.interpolate in fp64, rounded once.
"""
from collections import Counter

import torch
import torch.nn.functional as F

PSUM_LIMIT = 2 ** 20


def _dev(g):
    return g.device if isinstance(g, torch.Generator) else torch.device('cpu')


def int_acts(shape, g, amax=2):
    """integers in [-amax, amax] (fp32)"""
    return torch.randint(-amax, amax + 1, tuple(shape), generator=g, device=_dev(g)).float(), float(amax)


def int_weights(shape, g, density=1.0, l1max=None):
    """integers in {-1, 0, 1}, each kept with probability density; bound = largest L1 norm over dim 0 (outputs).
    l1max: keep only the first l1max non-zeros of each output (a hard bound, e.g. |main| <= 256 before a fused tail)"""
    w = torch.randint(-1, 2, tuple(shape), generator=g, device=_dev(g)).float()
    if density < 1.0:
        w = w * (torch.rand(tuple(shape), generator=g, device=_dev(g)) < density).float()
    if l1max is not None:
        f = w.flatten(1)
        f *= (f.abs().cumsum(1) <= l1max).float()
    return w, float(w.abs().flatten(1).sum(1).max().item())


def int_weights_convT(shape, g, density=1.0):
    """ConvTranspose weight [Cin, Cout, k, k]: bound = largest L1 norm over Cin of one (Cout, ky, kx) output"""
    w, _ = int_weights(shape, g, density)
    return w, float(w.abs().sum(0).max().item())


def int_bias(n, g, bmax=8):
    return torch.randint(-bmax, bmax + 1, (n,), generator=g, device=_dev(g)).float(), float(bmax)


def pow2(n, g, lo=-2, hi=2):
    """powers of two 2^k, k in [lo, hi]"""
    k = torch.randint(lo, hi + 1, (n,), generator=g, device=_dev(g)).float()
    return torch.exp2(k), float(2.0 ** hi)


def density_for(K, target_std=32.0, amax=2):
    """weight density that gives a K-term dot product of int_acts(amax) and int_weights an std of about target_std"""
    ea2 = sum(a * a for a in range(-amax, amax + 1)) / (2 * amax + 1)
    return min(1.0, target_std ** 2 / (K * ea2 * 2.0 / 3.0))


def psum_bound(amax, wl1, bmax=0.0, extra=0.0, scale=1.0):
    """bound on every partial sum of scale * (x . w) + bias (+ extra: residuals)"""
    return scale * amax * wl1 + bmax + extra


def check_bound(bound):
    assert bound <= PSUM_LIMIT, 'partial-sum bound %g exceeds 2^20: the probe would not be exact' % bound
    return bound


def is_bf16_exact(t):
    return bool((t.to(torch.bfloat16).double() == t.double()).all())


# ------------------------------------------------------------------------------------------------------ references
def round_to(ref64, dtype):
    """the one rounding of the fp64 reference to the kernel's output dtype"""
    return ref64.to(dtype)


def ref_linear(x, w, b=None):
    return F.linear(x.double(), w.double(), None if b is None else b.double())


def ref_conv(x, w, b=None, padding=None):
    padding = w.shape[-1] // 2 if padding is None else padding
    return F.conv2d(x.double(), w.double(), None if b is None else b.double(), padding=padding)


def ref_conv_transpose(x, w, b, k):
    return F.conv_transpose2d(x.double(), w.double(), None if b is None else b.double(), stride=k)


def ref_resize(x, size):
    """bilinear, align_corners=True, in fp64 (exact at dyadic ratios: the fractions are multiples of 1/4)"""
    return F.interpolate(x.double(), size=size, mode='bilinear', align_corners=True)


def dyadic_ratio(n_in, n_out):
    """align_corners scale (n_in - 1) / (n_out - 1), checked to be 1/2, 1/4 or 3/4 (or 1: no resample)"""
    r = (n_in - 1) / (n_out - 1)
    assert r in (0.25, 0.5, 0.75, 1.0), 'ratio %d -> %d is %g, not dyadic' % (n_in, n_out, r)
    return r


# ------------------------------------------------------------------------------------------------------ diagnosis
class Layout:
    """How output coordinates map to kernel tiles.
    kind 'rows': [rows, cols] token matrix, m-tiles of 128 rows.  kind 'nhwc': [NB, H, W, cols] map, pixel tiles of
    bh x bw.  Columns are logical output columns (col0 is added first), n-tiles of block_n."""

    def __init__(self, kind, block_n, bh=0, bw=0, col0=0, m_rows=128):
        assert kind in ('rows', 'nhwc')
        self.kind, self.block_n, self.bh, self.bw, self.col0, self.m_rows = kind, block_n, bh, bw, col0, m_rows

    @classmethod
    def from_desc(cls, d, col0=0):
        """from the pf_gemm descriptor ops.gemm returns (block_n, bh, bw filled in by the launch)"""
        if d.a_mode == 1:
            return cls('nhwc', d.block_n, d.bh, d.bw, col0)
        return cls('rows', d.block_n, col0=col0)

    def describe(self, idx, shape):
        """one mismatch coordinate -> (text, tile-relative position key, tile-relative column)"""
        col = idx[-1] + self.col0
        nt, ncol = col // self.block_n, col % self.block_n
        if self.kind == 'rows':
            row = idx[0]
            mt, r = row // self.m_rows, row % self.m_rows
            return ('(row %d, col %d): m-tile %d row %d (warp %d), n-tile %d col %d' % (row, col, mt, r, r // 16, nt, ncol),
                    'row %3d' % r, ncol)
        img, y, x = idx[0], idx[1], idx[2]
        H, W = shape[1], shape[2]
        tiles_y, tiles_x = (H + self.bh - 1) // self.bh, (W + self.bw - 1) // self.bw
        ty, tx = y // self.bh, x // self.bw
        mt = (img * tiles_y + ty) * tiles_x + tx
        ry, rx = y % self.bh, x % self.bw
        edge = []
        if y == 0 or y == H - 1:
            edge.append('top' if y == 0 else 'bottom')
        if x == 0 or x == W - 1:
            edge.append('left' if x == 0 else 'right')
        return ('(img %d, y %d, x %d, col %d): pixel tile (%d, %d) of %dx%d, m-tile %d, in-tile (%d, %d), n-tile %d col %d%s'
                % (img, y, x, col, ty, tx, self.bh, self.bw, mt, ry, rx, nt, ncol,
                   ' [image edge: %s]' % '/'.join(edge) if edge else ''),
                'in-tile (%2d, %3d)' % (ry, rx), ncol)


def mismatches(got, want):
    """boolean map of elements that differ (NaN anywhere in got counts; +0 and -0 are equal)"""
    g, w = got.double(), want.double()
    return (g != w) | torch.isnan(g) | torch.isnan(w)


def mismatch_report(got, want, layout, first=8, hist=8):
    """'' when got == want, else a report: count, the first coordinates with their tiles, and histograms of the
    mismatches by tile-relative position and tile-relative column"""
    bad = mismatches(got, want)
    n = int(bad.sum().item())
    if n == 0:
        return ''
    idx = bad.nonzero()[:20000].cpu().tolist()
    g, w = got.double().cpu(), want.double().cpu()
    lines = ['%d of %d elements differ (layout %s, block_n %d%s)' % (
        n, bad.numel(), layout.kind, layout.block_n,
        ', pixel tile %dx%d' % (layout.bh, layout.bw) if layout.kind == 'nhwc' else '')]
    pos, cols = Counter(), Counter()
    for i in idx[:20000]:                                   # histograms of the first 20000 (a Python loop)
        _, p, c = layout.describe(i, tuple(got.shape))
        pos[p] += 1
        cols[c] += 1
    for i in idx[:first]:
        text, _, _ = layout.describe(i, tuple(got.shape))
        lines.append('  %s: got %r want %r' % (text, g[tuple(i)].item(), w[tuple(i)].item()))
    lines.append('  by tile-relative position: ' + ', '.join('%s x%d' % kv for kv in pos.most_common(hist)))
    lines.append('  by tile-relative column:   ' + ', '.join('%d x%d' % kv for kv in cols.most_common(hist)))
    return '\n'.join(lines)


def assert_exact(name, got, want, layout):
    rep = mismatch_report(got, want, layout)
    assert not rep, '%s is not bit-exact:\n%s' % (name, rep)
