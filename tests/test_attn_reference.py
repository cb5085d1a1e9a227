"""CPU guard for the power of the pf_attention tests (no GPU needed).

test_gpu_attn_parity.py holds the kernel to FP64_TOL against an fp64 reference and to the ones-V invariant (V = 1 gives
1.0 within one bf16 ulp).  Here, on the CPU and at small shapes (one head, 128 query rows), the kernel-emulating
reference must stay inside those bounds in every softmax regime the GPU tests use, and emulations of three bugs the
suite exists to catch must fall outside them in the cases designed for each.  A later loosening of a bound that would
let one of these bugs through fails here.
"""
import pytest
import torch

from attn_ref import FP64_TOL, attention_emulated, attention_fp64, make_case, ones_v_error, per_head, rel_linf

REGIMES = [
    ('random', dict(std=0.3)), ('random', dict(std=1.0)), ('random', dict(std=8.0)), ('random', dict(std=30.0)),
    ('random', dict(std=8.0, via='magnitude')), ('random', dict(std=30.0, via='magnitude')),
    ('all_negative', {}), ('hot_last_key', {}), ('rising_max', {}), ('first_block_max', {}),
]


def _ids(cases):
    return ['%s%s' % (n, ''.join('-%s' % v for v in kw.values())) for n, kw in cases]


def _inputs(name, seq, kw, rows=128):
    q, k, v, scale = make_case(name, 1, seq, 1, seq, 'cpu', **kw)
    q, k, v = (per_head(t)[0, 0] for t in (q, k, v))
    return q[:rows], k, v, scale


@pytest.mark.parametrize('seq', [129, 1037])
@pytest.mark.parametrize('name,kw', REGIMES, ids=_ids(REGIMES))
def test_emulation_meets_the_gpu_bounds(seq, name, kw):
    q, k, v, scale = _inputs(name, seq, kw)
    err = rel_linf(attention_emulated(q, k, v, scale), attention_fp64(q, k, v, scale))
    print('%s seq %d: emulation vs fp64 rel-Linf %.2e' % (name, seq, err))
    assert err < FP64_TOL
    assert ones_v_error(attention_emulated(q, k, torch.ones_like(v), scale)) <= 1


# (bug, case, seq): each planted bug against the GPU cases built to expose it
CATCHERS = [
    ('mask_off_by_one', 'all_negative', 129), ('mask_off_by_one', 'all_negative', 1025),
    ('mask_off_by_one', 'all_negative', 1037),
    ('no_o_rescale', 'rising_max', 129), ('no_o_rescale', 'rising_max', 1037),
    ('l_counts_masked', 'all_negative', 129), ('l_counts_masked', 'all_negative', 1037),
    ('l_counts_masked', 'random', 129),
]


@pytest.mark.parametrize('bug,name,seq', CATCHERS)
def test_planted_bug_fails_the_gpu_bounds(bug, name, seq):
    q, k, v, scale = _inputs(name, seq, {})
    err = rel_linf(attention_emulated(q, k, v, scale, bug=bug), attention_fp64(q, k, v, scale))
    ones = ones_v_error(attention_emulated(q, k, torch.ones_like(v), scale, bug=bug))
    print('%s on %s seq %d: rel-Linf %.2e, ones-V %.1f ulp' % (bug, name, seq, err, ones))
    # a margin of 4x: the bug must not sit just above a bound that a small loosening would cross
    assert err > 4 * FP64_TOL
    assert ones > 4
