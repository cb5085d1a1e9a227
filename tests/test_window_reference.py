"""CPU guard for the Swin window-attention tests (no GPU needed).

test_gpu_window_attn.py holds pf_window_attention to the bounds in window_ref.py.  Here:
- the fp64 reference, the kernel emulation and pf_oracle.shift_mask match the reference's own G2LBasicLayer /
  SwinTransformerBlock outputs committed in tests/golden/window_case0.npz (oracle/make_golden_window.py);
- the emulation stays inside those bounds on small versions of every case family the GPU tests use;
- every planted bug lands at least 4x above its bound in a case built to catch it, so a later loosening of a bound
  that would let one of them through fails here.
"""
import os

import numpy as np
import pytest
import torch

import window_ref as wr

GOLD = os.path.join(os.path.dirname(__file__), 'golden', 'window_case0.npz')
# (H, W, C, heads, B) of the fixture
GEOMS = [(14, 19, 32, 8, 2), (14, 19, 64, 16, 1), (12, 30, 32, 8, 1), (12, 30, 64, 16, 1)]


@pytest.fixture(scope='module')
def gold():
    return {k: torch.from_numpy(v) for k, v in np.load(GOLD).items()}


def _crop(o, Hp, Wp, H, W):
    return o.reshape(o.shape[0], Hp, Wp, -1)[:, :H, :W].reshape(o.shape[0], H * W, -1)


@pytest.mark.parametrize('shift', [0, 6])
@pytest.mark.parametrize('H,W,C,heads,B', GEOMS)
def test_references_match_fixture(gold, H, W, C, heads, B, shift):
    t = '%dx%d_c%d' % (H, W, C)
    qkv, table = gold['qkv_' + t].float(), gold['table_' + t]
    want = gold['attn_%s_s%d' % (t, shift)]
    Hp, Wp = wr.padded(H, W)
    assert qkv.shape == (B, Hp * Wp, 3 * C) and torch.equal(wr.rb(qkv), qkv)
    ref = _crop(wr.window_attention_fp64(qkv, table, Hp, Wp, C, heads, shift), Hp, Wp, H, W)
    emu = _crop(wr.window_attention_emulated(qkv, table, Hp, Wp, C, heads, shift), Hp, Wp, H, W)
    e64, eemu = wr.rel_linf(want, ref), wr.rel_linf(emu, want)
    print('%s shift %d: fixture vs fp64 %.2e, emulation vs fixture %.2e' % (t, shift, e64, eemu))
    assert e64 <= 1e-6                    # the fixture is the reference in fp32
    assert eemu <= wr.FP64_TOL / 2
    # the shift and the mask matter here: without them, or with the other shift, the result is far from the fixture
    other = _crop(wr.window_attention_fp64(qkv, table, Hp, Wp, C, heads, 6 - shift), Hp, Wp, H, W)
    assert wr.rel_linf(other, want) > 4 * wr.FP64_TOL


@pytest.mark.parametrize('H,W', [(14, 19), (12, 30)])
def test_shift_mask_matches_fixture(gold, H, W):
    from oracle import pf_oracle as po
    Hp, Wp = wr.padded(H, W)
    cross = gold['mask_%dx%d' % (H, W)]
    assert torch.equal(po.shift_mask(Hp, Wp, 12, 'cpu') != 0, cross)
    # the kernel's region table gives the same cross-region pairs, window by window
    _, sreg = wr.kernel_tokens(Hp, Wp, 6)
    assert torch.equal(sreg[:, :, None] != sreg[:, None, :], cross)


def test_fixture_holds_reference_outputs_only(gold):
    names = {'qkv', 'table', 'attn', 'mask'}
    assert {k.split('_')[0] for k in gold} == names
    assert all(v.dtype in (torch.float16, torch.float32, torch.bool) for v in gold.values())


# ------------------------------------------------------------------------------------------------ emulations
# small versions of the GPU shapes: (H, W, C, heads), one per compiled head dim, and the grid edges
SMALL = [(14, 19, 32, 8), (24, 36, 64, 16), (12, 30, 16, 8), (13, 25, 256, 32), (12, 12, 16, 8), (14, 19, 8, 4),
         (25, 13, 16, 8)]


@pytest.mark.parametrize('shift', [0, 6])
@pytest.mark.parametrize('name', list(wr.CASES))
def test_emulation_meets_the_gpu_bounds(name, shift):
    worst = 0.0
    for i, (H, W, C, heads) in enumerate(SMALL[:4] if name in ('random', 'peaky') else SMALL[:2] + SMALL[4:]):
        Hp, Wp = wr.padded(H, W)
        qkv, table = wr.make_case(name, 2, H, W, C, heads, shift, seed=i)
        ref = wr.window_attention_fp64(qkv, table, Hp, Wp, C, heads, shift)
        emu = wr.window_attention_emulated(qkv, table, Hp, Wp, C, heads, shift)
        err = wr.rel_linf(emu, ref)
        worst = max(worst, err)
        print('%s shift %d %dx%d C%d h%d: emulation vs fp64 %.2e' % (name, shift, H, W, C, heads, err))
        if name == 'self_select':
            assert torch.equal(emu, wr.self_select_expected(2, Hp, Wp, C))
        if name == 'ones_v':
            assert ((emu - 1).abs() <= wr.bf16_ulp(torch.ones(1))).all()
    # the fp64 bound is twice the emulation's worst error: the emulation must stay at or below half of it
    assert worst <= wr.FP64_TOL / 2


# ------------------------------------------------------------------------------------------------ planted bugs
# (bug, case, shift, (H, W, C, heads))
CATCHERS = [
    ('mask_log2_domain', 'mask_dominance', 6, (14, 19, 32, 8)),
    ('mask_log2_domain', 'mask_dominance', 6, (12, 30, 16, 8)),
    ('region_off_by_one', 'mask_dominance', 6, (14, 19, 32, 8)),
    ('region_off_by_one', 'random', 6, (24, 36, 64, 16)),
    ('bias_transposed', 'offset_select', 0, (14, 19, 32, 8)),
    ('bias_transposed', 'offset_select', 6, (12, 12, 16, 8)),
    ('no_rescale', 'rising_max', 0, (14, 19, 32, 8)),
    ('no_rescale', 'hot_last_key', 6, (14, 19, 8, 4)),
    ('roll_backwards', 'random', 6, (14, 19, 32, 8)),
    ('roll_backwards', 'mask_dominance', 6, (12, 30, 16, 8)),
]


@pytest.mark.parametrize('bug,name,shift,shape', CATCHERS)
def test_planted_bug_fails_the_gpu_bound(bug, name, shift, shape):
    H, W, C, heads = shape
    Hp, Wp = wr.padded(H, W)
    qkv, table = wr.make_case(name, 1, H, W, C, heads, shift, seed=7)
    ref = wr.window_attention_fp64(qkv, table, Hp, Wp, C, heads, shift)
    got = wr.window_attention_emulated(qkv, table, Hp, Wp, C, heads, shift, bug=bug)
    err = wr.rel_linf(got, ref)
    emu = wr.window_attention_emulated(qkv, table, Hp, Wp, C, heads, shift)
    eemu = wr.emu_error(got, emu, qkv, C)
    print('%s on %s shift %d: %.2e vs fp64 (bound %.1e), %.1f x the emulation bound' % (bug, name, shift, err,
                                                                                       wr.FP64_TOL, eemu))
    assert err > 4 * wr.FP64_TOL
    assert eemu > 4


def test_random_inputs_miss_the_mask_bug():
    """why mask_dominance exists: with random logits a masked weight is negligible either way (e^-100 or e^-69)"""
    H, W, C, heads = 14, 19, 32, 8
    Hp, Wp = wr.padded(H, W)
    qkv, table = wr.make_case('random', 1, H, W, C, heads, 6, seed=7)
    ref = wr.window_attention_fp64(qkv, table, Hp, Wp, C, heads, 6)
    got = wr.window_attention_emulated(qkv, table, Hp, Wp, C, heads, 6, bug='mask_log2_domain')
    assert wr.rel_linf(got, ref) <= wr.FP64_TOL


def test_every_planted_bug_has_a_catcher():
    assert {c[0] for c in CATCHERS} == set(wr.PLANTED_BUGS)
