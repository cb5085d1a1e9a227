"""CPU checks of the bit-exact probe generators and of mismatch_report (tests/exact_ref.py)."""
import pytest
import torch
import torch.nn.functional as F

import exact_ref as er


def _g(seed):
    return torch.Generator().manual_seed(seed)


@pytest.mark.parametrize('K,density', [(32, 1.0), (592, 1.0), (4896, 1.0), (4896, er.density_for(4896)), (9 * 1088, 1.0)])
def test_generators_keep_their_bound(K, density):
    g = _g(K)
    x, amax = er.int_acts((64, K), g)
    w, wl1 = er.int_weights((48, K), g, density)
    b, bmax = er.int_bias(48, g)
    r, rmax = er.int_acts((64, 48), g)
    bound = er.check_bound(er.psum_bound(amax, wl1, bmax, extra=2 * rmax))
    assert x.abs().max() <= amax and w.abs().max() <= 1 and b.abs().max() <= bmax
    assert (x == x.round()).all() and (w == w.round()).all() and (b == b.round()).all()
    # the bound holds for every prefix of every dot product, not only the full sums
    prefix = (x[:, None, :] * w[None, :, :]).cumsum(-1).abs().max()
    assert prefix + bmax + 2 * rmax <= bound
    if density < 1.0:
        frac = (w != 0).float().mean().item()
        assert abs(frac - density * 2 / 3) < 0.02


def test_density_targets_small_outputs():
    """sparse weights keep a 3x3 conv over 544 channels mostly below 256, where bf16 holds every integer"""
    g = _g(1)
    K = 9 * 544
    x, _ = er.int_acts((256, K), g)
    w, _ = er.int_weights((64, K), g, er.density_for(K))
    y = x @ w.t()
    assert 20 < y.std() < 48
    assert (y.abs() < 256).float().mean() > 0.99


def test_powers_of_two():
    s, smax = er.pow2(100, _g(2), -3, 3)
    assert (torch.log2(s) == torch.log2(s).round()).all() and s.max() <= smax and s.min() >= 2 ** -3


def test_inputs_are_bf16_exact_and_pack_cannot_round_them():
    """every probe value survives the fp32 -> bf16 conversions (pf_pack_weight, the NHWC staging, the BN fold w * scale)"""
    g = _g(3)
    x, _ = er.int_acts((1000,), g)
    w, _ = er.int_weights((64, 600), g, 0.3)
    b, _ = er.int_bias(64, g)
    s, _ = er.pow2(64, g)
    r, _ = er.int_acts((1000,), g, amax=8)
    for t in (x, w, b, s, r, w * s[:, None], b * s):
        assert er.is_bf16_exact(t)
        assert torch.equal(t.to(torch.bfloat16).float(), t)
    # a value that is not bf16-exact is caught
    assert not er.is_bf16_exact(torch.tensor([1.0 + 2 ** -10]))


def test_dyadic_resample_is_bf16_exact():
    """align_corners ratios of 1/2, 1/4 and 3/4 put every source coordinate on a multiple of 1/4: the resampled
    integers are multiples of 1/16 and survive the kernel's bf16 rounding"""
    g = _g(4)
    for (h, w), (H, W) in [((13, 19), (25, 37)), ((7, 10), (25, 37)), ((25, 37), (33, 49))]:
        er.dyadic_ratio(h, H)
        er.dyadic_ratio(w, W)
        x, _ = er.int_acts((2, 8, h, w), g)
        up = er.ref_resize(x, (H, W))
        assert er.is_bf16_exact(up)
        assert ((up * 16) == (up * 16).round()).all()
        # the fp32 torch resample agrees with fp64 bit for bit
        assert torch.equal(F.interpolate(x, size=(H, W), mode='bilinear', align_corners=True).double(), up)
    with pytest.raises(AssertionError):
        er.dyadic_ratio(35, 40)


@pytest.mark.parametrize('case', ['linear', 'conv3', 'convT', 'resample'])
def test_fp64_reference_equals_fp32(case):
    """exactness does not depend on summation order: fp32 on the CPU gives the fp64 result bit for bit"""
    g = _g(5)
    if case == 'linear':
        x, _ = er.int_acts((300, 592), g)
        w, _ = er.int_weights((200, 592), g)
        b, _ = er.int_bias(200, g)
        r64, r32 = er.ref_linear(x, w, b), F.linear(x, w, b)
    elif case == 'conv3':
        x, _ = er.int_acts((2, 136, 13, 11), g)
        w, _ = er.int_weights((40, 136, 3, 3), g)
        b, _ = er.int_bias(40, g)
        r64, r32 = er.ref_conv(x, w, b), F.conv2d(x, w, b, padding=1)
    elif case == 'convT':
        x, _ = er.int_acts((2, 72, 5, 7), g)
        w, _ = er.int_weights_convT((72, 32, 4, 4), g)
        b, _ = er.int_bias(32, g)
        r64, r32 = er.ref_conv_transpose(x, w, b, 4), F.conv_transpose2d(x, w, b, stride=4)
    else:
        x, _ = er.int_acts((2, 24, 7, 10), g)
        w, _ = er.int_weights((16, 24, 3, 3), g)
        up = er.ref_resize(x, (25, 37))
        r64 = er.ref_conv(up, w)
        r32 = F.conv2d(F.interpolate(x, size=(25, 37), mode='bilinear', align_corners=True), w, padding=1)
    assert torch.equal(r64, r32.double())
    assert torch.equal(er.round_to(r64, torch.bfloat16), r32.to(torch.bfloat16))


def test_mismatch_report_names_the_tile_nhwc():
    g = _g(6)
    want = er.int_acts((3, 21, 13, 40), g)[0].to(torch.bfloat16)
    got = want.clone()
    assert er.mismatch_report(got, want, er.Layout('nhwc', 32, 16, 8)) == ''
    got[2, 17, 9, 35] += 1                          # image 2, pixel tile (1, 1) of 2 x 2, in-tile (1, 1), n-tile 1
    rep = er.mismatch_report(got, want, er.Layout('nhwc', 32, 16, 8))
    assert rep.startswith('1 of %d elements differ' % want.numel())
    assert '(img 2, y 17, x 9, col 35): pixel tile (1, 1) of 16x8, m-tile 11, in-tile (1, 1), n-tile 1 col 3' in rep
    assert 'in-tile ( 1,   1) x1' in rep
    got[0, 0, 12, 0] = float('nan')                 # NaN counts, at an image corner
    rep = er.mismatch_report(got, want, er.Layout('nhwc', 32, 16, 8))
    assert rep.startswith('2 of') and 'image edge: top/right' in rep
    with pytest.raises(AssertionError, match='not bit-exact'):
        er.assert_exact('probe', got, want, er.Layout('nhwc', 32, 16, 8))


def test_mismatch_report_names_the_tile_rows():
    g = _g(7)
    want = er.int_acts((300, 200), g)[0]
    got = want.clone()
    got[130:300:16, 199] -= 2                       # a column of errors in the last n-tile, one row per warp
    rep = er.mismatch_report(got, want, er.Layout('rows', 96, col0=8))
    assert rep.startswith('11 of 60000 elements differ')
    assert '(row 130, col 207): m-tile 1 row 2 (warp 0), n-tile 2 col 15' in rep
    assert 'by tile-relative column:   15 x11' in rep
    # +0 and -0 are the same value
    z = torch.zeros(4, 4)
    assert er.mismatch_report(-z, z, er.Layout('rows', 32)) == ''
