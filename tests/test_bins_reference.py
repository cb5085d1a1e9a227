"""CPU guard for the metric-bins tail tests (no GPU needed).

test_gpu_bins_tail.py holds pf_attractor, pf_logbinom_depth and pf_add_upsampled to the bounds in bins_ref.py.  Here:
- the fp64 references and the oracle's fp32 restatement, including the exp / sum modes no shipped config uses, match
  the reference layers' outputs committed in tests/golden/bins_case0.npz (oracle/make_golden_bins.py);
- the kernel emulations stay inside those bounds in every regime the GPU tests use;
- every planted bug lands at least 4x above its bound in a case built to catch it, so a later loosening of a bound
  that would let one of them through fails here.
"""
import os

import numpy as np
import pytest
import torch

import bins_ref as br

GOLD = os.path.join(os.path.dirname(__file__), 'golden', 'bins_case0.npz')
LB_SHAPE = (1, (28, 37), (49, 65))          # bins h x w -> depth H x W (non-dyadic), small enough for the CPU


@pytest.fixture(scope='module')
def gold():
    return {k: torch.from_numpy(v) for k, v in np.load(GOLD).items()}


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize('nA', [16, 4, 1])
@pytest.mark.parametrize('flags', range(4))
def test_attractor_references_match_fixture(gold, flags, nA):
    from oracle import pf_oracle as po
    kind, typ = br.ATTRACTOR_FLAGS[flags]
    want = gold['att_%s_%s_%d' % (kind, typ, nA)]
    A, b_prev = gold['att_A'][:, :nA].contiguous(), gold['att_b_prev']
    ref, delta = br.attractor_fp64(_nhwc(A), nA, _nhwc(b_prev), kind, typ)
    e64 = br.rel_linf(_nhwc(want), ref)
    e32 = br.rel_linf(po.attractor_update(A, b_prev, kind, typ), want)
    # the fixture is the reference in fp32: a few ulps of |b| from fp64 (chain bound), and the oracle's same ops
    print('%s/%s nA %d: fp64 vs fixture %.2e, oracle vs fixture %.2e, max|delta| %.2e' % (kind, typ, nA, e64, e32,
                                                                                       delta.abs().max()))
    assert e64 <= br.chain_tol(*b_prev.shape[-2:])
    assert e32 <= 1e-7
    # the mode matters in this case: every other (kind, type) pair is far from the fixture (for one attractor the mean
    # is the sum)
    for other in range(4):
        okind, otyp = br.ATTRACTOR_FLAGS[other]
        if other == flags or (nA == 1 and otyp == typ):
            continue
        o = br.attractor_fp64(_nhwc(A), nA, _nhwc(b_prev), okind, otyp)[0]
        assert br.rel_linf(_nhwc(want), o) > 4 * br.chain_tol(*b_prev.shape[-2:]), (okind, otyp)


@pytest.mark.parametrize('regime', ['mid', 'sharp', 'flat', 'p_low', 'q_low'])
def test_logbinom_references_match_fixture(gold, regime):
    pt, bc = _nhwc(gold['lb_pt_' + regime]), _nhwc(gold['lb_bc'])
    want = gold['lb_depth_' + regime]
    H, W = want.shape[-2:]
    ref = br.logbinom_depth_fp64(pt, bc, H, W)
    o32 = br.logbinom_depth_oracle32(pt, bc, H, W)
    e64, e32 = br.rel_linf(want, ref), br.rel_linf(o32, want)
    print('%s: fixture vs fp64 %.2e, oracle vs fixture %.2e' % (regime, e64, e32))
    assert e64 <= br.logbinom_tol(br.rel_linf(o32, ref))
    assert e32 == 0.0


# ------------------------------------------------------------------------------------------------ emulations
# (family, level, sigma); sigma None: attractors far from every bin
ATT_CASES = [('chain', 0, 0.02), ('chain', 0, 0.2), ('chain', 1, 0.06), ('exact', 0, 0.02), ('exact', 0, 0.06),
             ('exact', 1, 0.2), ('exact', 2, 0.06), ('exact', 0, None)]


def _attractor_err(family, A, nA, b_prev, flags, bug=None):
    kind, typ = br.ATTRACTOR_FLAGS[flags]
    ref, delta = br.attractor_fp64(A, nA, b_prev, kind, typ)
    got = br.attractor_emulated(A, nA, b_prev, flags, bug)
    if family == 'exact':
        return br.attractor_exact_error(got, ref, delta), br.ATT_EXACT_TOL
    return br.rel_linf(got, ref), br.chain_tol(*b_prev.shape[1:3])


@pytest.mark.parametrize('family,level,sigma', ATT_CASES)
def test_attractor_emulation_meets_the_gpu_bounds(family, level, sigma):
    hw, HW, nA = (br.CHAIN if family == 'chain' else br.EXACT_CHAIN)[level]
    A, b_prev = br.attractor_case(2, hw, HW, nA, torch.Generator().manual_seed(level), family, sigma=sigma or 0,
                                  far=sigma is None)
    for flags in range(4):
        err, tol = _attractor_err(family, A, nA, b_prev, flags)
        print('%s level %d sigma %s flags %d: %.2e (bound %.2e)' % (family, level, sigma, flags, err, tol))
        assert err <= tol / 4


@pytest.mark.parametrize('regime', br.REGIMES)
def test_logbinom_emulation_meets_the_gpu_bounds(regime):
    B, bhw, HW = LB_SHAPE
    pt, bc = br.logbinom_case(B, bhw, HW, regime, torch.Generator().manual_seed(1))
    ref = br.logbinom_depth_fp64(pt, bc, *HW)
    tol = br.logbinom_tol(br.rel_linf(br.logbinom_depth_oracle32(pt, bc, *HW), ref))
    err = br.rel_linf(br.logbinom_depth_emulated(pt, bc, *HW), ref)
    print('%s: emulation %.2e (bound %.2e)' % (regime, err, tol))
    assert err <= tol


@pytest.mark.parametrize('level', [0, 1])
def test_add_upsampled_emulation_meets_the_gpu_bound(level):
    hw, HW, _ = br.CHAIN[level]
    a, prev = br.add_upsampled_case(2, hw, HW, 128, torch.Generator().manual_seed(level))
    err = br.add_upsampled_error(br.add_upsampled_emulated(a, prev), a, prev)
    print('level %d: %.2f of the bound' % (level, err))
    assert err <= 1.0


# ------------------------------------------------------------------------------------------------ planted bugs
# (bug, family, (h, w) -> (H, W), nA, flags, sigma, B)
ATT_CATCHERS = [
    ('align_corners_false', 'chain', ((14, 19), (28, 37)), 16, 1, 0.06, 2),
    ('mean_sum_swapped', 'exact', ((15, 19), (29, 37)), 16, 1, 0.06, 2),
    ('mean_sum_swapped', 'exact', ((15, 19), (29, 37)), 16, 2, 0.06, 2),
    ('inv_exp_swapped', 'exact', ((15, 19), (29, 37)), 16, 1, 0.02, 2),
    ('inv_exp_swapped', 'exact', ((15, 19), (29, 37)), 1, 2, 0.06, 2),
    ('image0_only', 'chain', ((14, 19), (28, 37)), 16, 1, 0.06, 3),
    ('hi_unclamped', 'chain', ((28, 37), (28, 37)), 16, 1, 0.06, 3),
    ('hi_unclamped', 'chain', ((1, 19), (28, 37)), 16, 1, 0.06, 3),
    ('no_mean_divide', 'exact', ((29, 37), (57, 73)), 8, 3, 0.06, 2),
]


@pytest.mark.parametrize('bug,family,sizes,nA,flags,sigma,B', ATT_CATCHERS)
def test_attractor_planted_bug_fails_the_gpu_bound(bug, family, sizes, nA, flags, sigma, B):
    A, b_prev = br.attractor_case(B, *sizes, nA, torch.Generator().manual_seed(7), family, sigma=sigma)
    err, tol = _attractor_err(family, A, nA, b_prev, flags, bug)
    print('%s: %.2e (bound %.2e)' % (bug, err, tol))
    assert err > 4 * tol


LB_CATCHERS = [('p_clamp_dropped', 'p_low'), ('p_clamp_dropped', 'mix'), ('q_clamp_dropped', 'q_low'),
               ('temp_multiplied', 'mid'), ('temp_multiplied', 'sharp'), ('bins_reversed', 'mid'),
               ('bins_reversed', 'sharp'), ('no_butterfly', 'mid'), ('no_butterfly', 'flat'),
               ('butterfly_two_steps', 'mid'), ('bins_scale', 'mid')]


@pytest.mark.parametrize('bug,regime', LB_CATCHERS)
def test_logbinom_planted_bug_fails_the_gpu_bound(bug, regime):
    B, bhw, HW = LB_SHAPE
    pt, bc = br.logbinom_case(B, bhw, HW, regime, torch.Generator().manual_seed(3))
    ref = br.logbinom_depth_fp64(pt, bc, *HW)
    tol = br.logbinom_tol(br.rel_linf(br.logbinom_depth_oracle32(pt, bc, *HW), ref))
    err = br.rel_linf(br.logbinom_depth_emulated(pt, bc, *HW, bug=bug), ref)
    print('%s on %s: %.2e (bound %.2e)' % (bug, regime, err, tol))
    assert err > 4 * tol


def test_add_upsampled_planted_bug_fails_the_gpu_bound():
    a, prev = br.add_upsampled_case(2, (14, 19), (28, 37), 128, torch.Generator().manual_seed(5))
    err = br.add_upsampled_error(br.add_upsampled_emulated(a, prev, bug='align_corners_false'), a, prev)
    print('align_corners_false: %.1f x the bound' % err)
    assert err > 4


def test_every_planted_bug_has_a_catcher():
    caught = {('attractor', c[0]) for c in ATT_CATCHERS} | {('logbinom', c[0]) for c in LB_CATCHERS}
    caught.add(('add_upsampled', 'align_corners_false'))
    assert caught == {(k, b) for k, bugs in br.PLANTED_BUGS.items() for b in bugs}
