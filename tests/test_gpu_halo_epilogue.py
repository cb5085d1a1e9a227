"""The bulk-store epilogue of pf_conv3_halo_kernel on bit-exact integer probes (tests/exact_ref.py).

Plain bf16 outputs of the halo kernel are finished in the accumulator's fragment layout, staged with stmatrix and
stored as {64 or 32 channels, 8 px, 2 rows} boxes.  The probes cover every halo width (N = 544 ends in a 64-column group
with 32 valid columns), images whose sides are not multiples of the 16 x 8 pixel tile, odd tile counts under clusters
of 2 and 4 CTAs (the phantom tile past the last image), outputs inside a wider buffer (out_col0 > 0, out_ld > N) whose
other columns hold a poison value that must survive, and ReLU or no activation.  Each case must equal the fp64
reference rounded once and the row-per-thread epilogue (PF_OPT_TMA_EPILOGUE = 0) bit for bit.
"""
import zlib

import pytest
import torch
import torch.nn.functional as F

import exact_ref as er
from exact_ref import Layout, assert_exact

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

POISON = -7.0


def _gen(*key):
    return torch.Generator(device='cuda').manual_seed(zlib.crc32(repr(key).encode()))


def _run(pw, src, NB, H, W, N, act, col0, ld, tma, cluster):
    from patchfusion_b200 import lib, ops
    out = torch.full((NB, H, W, ld), POISON, dtype=torch.bfloat16, device='cuda')
    lib.call('pf_set_option', lib.OPT_TMA_EPILOGUE, tma)
    lib.call('pf_set_option', lib.OPT_HALO_MULTICAST, cluster)
    try:
        d = ops.gemm(pw, [src], out, image=(NB, H, W), act=act, out_col0=col0)
        torch.cuda.synchronize()
    finally:
        lib.call('pf_set_option', lib.OPT_TMA_EPILOGUE, 1)
        lib.call('pf_set_option', lib.OPT_HALO_MULTICAST, 1)
    return d, out


# (N, Cin, block_n): every halo width; 544 = 192 + 192 + 160 and 768 = 4 x 192 as in the Guided-Fusion decoder
WIDTHS = [(32, 40, 32), (64, 64, 64), (128, 72, 128), (192, 136, 192), (544, 96, 192), (768, 64, 192)]
# (NB, H, W, cluster option 0 / 1 / 2 = CTAs of 1 / 2 / 4): every side ends inside a 16 x 8 pixel tile.  Clusters form
# once the tiles fill the GPU (>= 132 work items); 5 x 3 x 9 = 135 pixel tiles leave the last cluster of 2 or 4 with
# phantom tiles past the last image, 7 x 4 x 10 = 280 fill clusters of 4 exactly
GEOMS = [(3, 25, 37, 0), (5, 37, 71, 1), (5, 37, 71, 2), (7, 49, 73, 2)]


@pytest.mark.parametrize('N,cin,bn', WIDTHS)
@pytest.mark.parametrize('NB,H,W,cluster', GEOMS)
@pytest.mark.parametrize('relu', [True, False])
@pytest.mark.parametrize('col0,extra', [(0, 0), (24, 40)])
def test_halo_bulk_store_epilogue(cuda, N, cin, bn, NB, H, W, cluster, relu, col0, extra):
    from patchfusion_b200 import ops
    g = _gen('halo-epi', N, NB, H, W, relu, col0)
    x, amax = er.int_acts((NB, cin, H, W), g)
    wt, wl1 = er.int_weights((N, cin, 3, 3), g, er.density_for(9 * cin))
    b, bmax = er.int_bias(N, g)
    er.check_bound(er.psum_bound(amax, wl1, bmax))
    pw = ops.pack_weight(wt, b)
    src = x.permute(0, 2, 3, 1).to(torch.bfloat16).contiguous()
    ref = er.ref_conv(x, wt, b, padding=1)
    if relu:
        ref = F.relu(ref)
    ld = col0 + N + extra
    want = torch.full((NB, H, W, ld), POISON, dtype=torch.bfloat16, device='cuda')
    want[..., col0:col0 + N] = er.round_to(ref, torch.bfloat16).permute(0, 2, 3, 1)
    act = ops.ACT_RELU if relu else ops.ACT_NONE
    d, out = _run(pw, src, NB, H, W, N, act, col0, ld, 1, cluster)
    assert (d.block_n, d.bh, d.bw) == (bn, 16, 8)      # the halo kernel's 16 x 8 pixel tile
    name = 'halo N %d BN %d %dx%dx%d cl-opt %d relu %d col0 %d ld %d' % (N, bn, NB, H, W, cluster, relu, col0, ld)
    assert_exact(name, out, want, Layout.from_desc(d, col0=-col0))
    _, out0 = _run(pw, src, NB, H, W, N, act, col0, ld, 0, cluster)
    assert torch.equal(out.view(torch.int16), out0.view(torch.int16)), name + ': bulk-store and row-per-thread differ'
