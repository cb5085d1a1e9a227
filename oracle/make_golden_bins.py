"""Pins the metric-bins tail of oracle/pf_oracle.py (attractor_update, log_binomial_depth) against the reference's own
layers and writes tests/golden/bins_case0.npz.   python -m oracle.make_golden_bins  (needs $PATCHFUSION_REFERENCE)

- AttractorLayerUnnormed (memory_efficient=True, as in the configs) with its MLP replaced by nn.Identity(), so that
  the attractor points A are an input: every (kind, type) pair at nA = 16, 4, 1, B = 2, bin centres up-sampled at a
  non-dyadic ratio (5 x 6 -> 8 x 9).  Attractors sit near bin centres (N(0, 0.06)) so the shift is not negligible.
- ConditionalLogBinomial(4, 0, 64, min_temp=0.0212, max_temp=50) with its MLP replaced by nn.Identity(), on five
  (p, t) regimes (mid, t -> min_temp, t -> max_temp, p < 1e-4, 1 - p < 1e-4), followed by the expectation over the
  up-sampled bin centres (zoedepth_v1.py:214-219).
"""
import os
import sys

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import pf_oracle as po           # noqa: E402
from oracle import ref_harness as rh         # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden', 'bins_case0.npz')
B, NBINS, SRC, DST = 2, 64, (5, 6), (8, 9)
N_ATTRACTORS = (16, 4, 1)
PAIRS = (('mean', 'inv'), ('sum', 'inv'), ('mean', 'exp'), ('sum', 'exp'))
REGIMES = ('mid', 'sharp', 'flat', 'p_low', 'q_low')
MIN_TEMP, MAX_TEMP = 0.0212, 50.0


def case_inputs():
    g = torch.Generator().manual_seed(0)
    b_prev = torch.sort(1e-3 + torch.rand(B, NBINS, *SRC, generator=g) * 80, dim=1).values
    bu = F.interpolate(b_prev, DST, mode='bilinear', align_corners=True)
    k = torch.randint(0, NBINS, (B, max(N_ATTRACTORS), *DST), generator=g)
    A = torch.gather(bu, 1, k) + 0.06 * torch.randn(B, max(N_ATTRACTORS), *DST, generator=g)
    sp = lambda: F.softplus(torch.randn(B, 1, *DST, generator=g))               # noqa: E731
    big = lambda: 1e3 * (1 + torch.rand(B, 1, *DST, generator=g))               # noqa: E731
    zero = torch.zeros(B, 1, *DST)
    pt = {'mid': (sp(), sp(), sp(), sp()), 'sharp': (sp(), sp(), zero, big()), 'flat': (sp(), sp(), big(), zero),
          'p_low': (zero, 10 * big(), sp(), sp()), 'q_low': (10 * big(), zero, sp(), sp())}
    pt = {r: torch.cat(pt[r], 1) for r in REGIMES}
    bc = torch.sort(1e-3 + torch.rand(B, NBINS, *SRC, generator=g) * 80, dim=1).values
    return dict(att_A=A, att_b_prev=b_prev, lb_bc=bc, **{'lb_pt_' + r: pt[r] for r in REGIMES})


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()


def main():
    rh._enter()
    from zoedepth.models.layers.attractor import AttractorLayerUnnormed
    from zoedepth.models.layers.dist_layers import ConditionalLogBinomial
    x = case_inputs()
    out = {k: v.numpy() for k, v in x.items()}
    with torch.no_grad():
        for kind, typ in PAIRS:
            for nA in N_ATTRACTORS:
                layer = AttractorLayerUnnormed(8, NBINS, nA, kind=kind, attractor_type=typ, memory_efficient=True)
                layer._net = nn.Identity()
                A = x['att_A'][:, :nA].contiguous()
                ref, _ = layer(A, x['att_b_prev'])
                mine = po.attractor_update(A, x['att_b_prev'], kind, typ)
                e = _rel(mine, ref)
                print('attractor %s/%s nA %d: oracle vs reference rel-Linf %.2e' % (kind, typ, nA, e))
                assert e <= 1e-6, (kind, typ, nA, e)
                out['att_%s_%s_%d' % (kind, typ, nA)] = ref.numpy()
        clb = ConditionalLogBinomial(4, 0, NBINS, min_temp=MIN_TEMP, max_temp=MAX_TEMP)
        clb.mlp = nn.Identity()
        for r in REGIMES:
            pt = x['lb_pt_' + r]
            prob = clb(pt, torch.zeros(B, 0, *DST))
            ref = torch.sum(prob * F.interpolate(x['lb_bc'], DST, mode='bilinear', align_corners=True), 1)
            mine = po.log_binomial_depth(pt, x['lb_bc'], MIN_TEMP, MAX_TEMP)[:, 0]
            e = _rel(mine, ref)
            print('log-binomial depth %s: oracle vs reference rel-Linf %.2e' % (r, e))
            assert e <= 1e-6, (r, e)
            out['lb_depth_' + r] = ref.numpy()
    np.savez_compressed(OUT, **out)
    print('wrote', OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
