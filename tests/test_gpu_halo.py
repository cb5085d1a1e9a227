"""Halo-tile 3x3 conv at every compiled n-tile width (block_n 32 / 64 / 128 / 192), against torch fp32 on the same
bf16-rounded operands.

Each width is run with a zero-padded last n-tile where one exists, sources whose last 64-channel chunk is partial,
fused-resample sources, and weight-multicast clusters of 1, 2 and 4 CTAs.  Output columns beyond N must keep what
was there, and two identical launches must give identical bits.
"""
import pytest
import torch
import torch.nn.functional as F

from gpu_util import check, from_nhwc, rb, to_nhwc

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

SENTINEL = 3.0


def _run(cuda, NB, H, W, srcs, N, cluster, tail=None):
    """srcs: [(h, w, channels)]; a source of another size than (H, W) is read through the fused bilinear resample."""
    from patchfusion_b200 import lib, ops
    g = torch.Generator(device='cuda').manual_seed(H * W + N + len(srcs))
    cs = [c for _, _, c in srcs]
    xs = [torch.randn(NB, c, h, w, device=cuda, generator=g) for h, w, c in srcs]
    wt = torch.randn(N, sum(cs), 3, 3, device=cuda, generator=g) / (9 * sum(cs)) ** 0.5
    b = torch.randn(N, device=cuda, generator=g)
    pw = ops.pack_weight(wt, b, src_c=cs)
    resample = [(h, w) != (H, W) for h, w, _ in srcs]
    ld = ops.pad_to(N, 8) + 8
    kw = {}
    if tail is not None:
        n2 = tail
        w2 = torch.randn(n2, N, device=cuda, generator=g) / N ** 0.5
        b2 = torch.randn(n2, device=cuda, generator=g)
        kw = dict(tail=(w2, b2, ops.ACT_NONE))
    lib.call('pf_set_option', lib.OPT_HALO_MULTICAST, cluster)
    try:
        outs, descs, tails = [], [], []
        for _ in range(2):
            out = torch.full((NB, H, W, ld), SENTINEL, dtype=torch.bfloat16, device=cuda)
            if tail is not None:
                kw['tail_out'] = torch.zeros(NB, H, W, 16, dtype=torch.float32, device=cuda)
                tails.append(kw['tail_out'])
            descs.append(ops.gemm(pw, [to_nhwc(x) for x in xs], out, image=(NB, H, W), act=ops.ACT_RELU,
                                  resample=resample, **kw))
            outs.append(out)
        torch.cuda.synchronize()
    finally:
        lib.call('pf_set_option', lib.OPT_HALO_MULTICAST, 1)
    up = [rb(F.interpolate(rb(x), size=(H, W), mode='bilinear', align_corners=True)) if r else rb(x)
          for x, r in zip(xs, resample)]
    ref = F.relu(F.conv2d(torch.cat(up, 1), rb(wt), b, padding=1))
    name = 'halo %s -> %d @%dx%d cl-opt %d' % (srcs, N, H, W, cluster)
    check(name, from_nhwc(outs[0], N), ref, 1e-2)
    assert (outs[0][..., N:] == SENTINEL).all(), 'columns beyond N were written'
    assert torch.equal(outs[0], outs[1]), 'two identical launches differ'
    if tail is not None:
        tref = F.conv2d(ref, w2.view(n2, N, 1, 1), b2)
        check(name + ' tail', tails[0][..., :n2].permute(0, 3, 1, 2), tref, 2e-3)
        assert torch.equal(tails[0], tails[1])
    return descs[0]


# (N, expected block_n, n-tiles): 544 = 3 x 192 with 32 padded columns, 768 = 4 x 192, 256 = 2 x 128,
# 56 = 1 x 64 with 8 padded columns, 96 = 3 x 32, 32 = 1 x 32
@pytest.mark.parametrize('cs,N,bn,nt', [([32, 256, 256], 544, 192, 3), ([64], 768, 192, 4), ([40, 64], 256, 128, 2),
                                        ([96], 56, 64, 1), ([8], 96, 32, 3), ([136], 32, 32, 1)])
@pytest.mark.parametrize('cluster', [0, 1, 2])
def test_halo_block_n(cuda, cs, N, bn, nt, cluster):
    # 5 x 50 x 70: 180 pixel tiles (partial at the right and bottom edges), enough for the multicast clusters
    NB, H, W = 5, 50, 70
    d = _run(cuda, NB, H, W, [(H, W, c) for c in cs], N, cluster)
    assert (d.block_n, d.n_tiles) == (bn, nt)


@pytest.mark.parametrize('cluster', [0, 1, 2])
def test_halo_resample_block_n_192(cuda, cluster):
    NB, H, W = 5, 50, 70
    d = _run(cuda, NB, H, W, [(25, 35, 136), (H, W, 64), (37, 52, 40)], 544, cluster)
    assert d.block_n == 192


def test_halo_fused_tail_block_n_192(cuda):
    """fused trailing layer over a 192-column row: the two half-row partial sums meet in a warp shuffle"""
    d = _run(cuda, 2, 30, 41, [(30, 41, 64)], 192, 0, tail=4)
    assert (d.block_n, d.n_tiles) == (192, 1)


def test_halo_fused_tail_needs_one_tile(cuda):
    from patchfusion_b200 import lib
    with pytest.raises(lib.PFError, match='one N tile'):
        _run(cuda, 1, 16, 16, [(16, 16, 64)], 256, 0, tail=4)
