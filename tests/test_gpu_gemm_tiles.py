"""pf_gemm_kernel at every compiled n-tile width (block_n 32 / 64 / 96 / 128 / 192 / 256), against torch fp32 on the
same bf16-rounded operands.

Each width runs with a zero-padded last n-tile, K not a multiple of 64 (the patch embed's 592), the bf16 bulk-store
and the fp32 bulk reduce-add epilogues, with and without weight-multicast pairs.  Output columns beyond N must keep
what was there, and two identical launches must give identical bits.  Further cases: V^T and bulk-store tiles mixed in
one CTA, pixel shuffle, fused trailing layers at their width, 1x1 convs at every pixel-tile shape (4-D output boxes)
and the pinned-tile 3x3 path.
"""
import pytest
import torch
import torch.nn.functional as F

from gpu_util import bf, check, from_nhwc, rb, to_nhwc

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

SENTINEL = 3.0


def _lib_ops():
    from patchfusion_b200 import lib, ops
    return lib, ops


def _multicast(lib, on):
    lib.call('pf_set_option', lib.OPT_GEMM_MULTICAST, on)


# (M, N, expected block_n, n-tiles): N = 1000 sits in a 1024-row panel; 66 m-tiles are 4 waves of 128-column tiles on
# 132 SMs and 2 of 256-column ones (-> 256), 73 m-tiles are 5 against 3 (-> 128).  544 -> 576 rows = 3 x 192,
# 80 -> 96, 48 -> 64, 150 -> 160 = 5 x 32.
WIDTH_CASES = [(8398, 1000, 256, 4), (9333, 1000, 128, 8), (4144, 544, 192, 3), (20000, 80, 96, 1), (20000, 48, 64, 1),
               (9333, 150, 32, 5)]


@pytest.mark.parametrize('M,N,bn,nt', WIDTH_CASES)
@pytest.mark.parametrize('mode', ['bf16', 'gamma'])
@pytest.mark.parametrize('multicast', [0, 1])
def test_linear_block_n(cuda, M, N, bn, nt, mode, multicast):
    lib, ops = _lib_ops()
    if torch.cuda.get_device_properties(0).multi_processor_count != 132 and bn in (128, 256):
        pytest.skip('the 128 / 256 choice depends on the SM count (132 on an H100 SXM)')
    K = 592
    g = torch.Generator(device='cuda').manual_seed(M + N)
    x = torch.randn(M, K, device=cuda, generator=g)
    w = torch.randn(N, K, device=cuda, generator=g) / K ** 0.5
    b = torch.randn(N, device=cuda, generator=g)
    pw = ops.pack_weight(w, b)
    xa = bf(x).contiguous()
    ref = F.linear(rb(x), rb(w), b)
    ld = ops.pad_to(N, 8) + 8
    _multicast(lib, multicast)
    try:
        outs = []
        for _ in range(2):
            if mode == 'bf16':
                out = torch.full((M, ld), SENTINEL, dtype=torch.bfloat16, device=cuda)
                d = ops.gemm(pw, [xa], out, act=ops.ACT_GELU)
            else:
                gam = torch.rand(N, device=cuda, generator=torch.Generator(device='cuda').manual_seed(N))
                out = torch.full((M, ld), SENTINEL, dtype=torch.float32, device=cuda)
                d = ops.gemm(pw, [xa], out, gamma=gam)
            outs.append(out)
        torch.cuda.synchronize()
    finally:
        _multicast(lib, 1)
    name = 'linear %dx%dx%d %s bn %d mc %d' % (M, K, N, mode, bn, multicast)
    if mode == 'bf16':
        check(name, outs[0][:, :N], F.gelu(ref), 1e-2)
    else:
        check(name, outs[0][:, :N], SENTINEL + gam * ref, 2e-5)
    assert (outs[0][:, N:] == SENTINEL).all(), 'columns beyond N were written'
    assert torch.equal(outs[0], outs[1]), 'two identical launches differ'
    assert (d.block_n, d.n_tiles) == (bn, nt)


@pytest.mark.parametrize('D,seq,bn', [(384, 1500, 128), (768, 1400, 256)])
@pytest.mark.parametrize('multicast', [0, 1])
def test_qkv_vt_mixed_block_n(cuda, D, seq, bn, multicast):
    """Fused qkv projection whose n-tile count (9) does not divide the SM count: every CTA runs q/k tiles (bulk store)
    and V^T tiles (direct transposing store) one after the other."""
    lib, ops = _lib_ops()
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip('tile counts chosen for 132 SMs')
    g = torch.Generator(device='cuda').manual_seed(D + seq)
    B, K = 4, 64
    seq_pad = ops.pad_to(seq, 8)
    x = torch.randn(B * seq, K, device=cuda, generator=g)
    w = torch.randn(3 * D, K, device=cuda, generator=g) / K ** 0.5
    b = torch.randn(3 * D, device=cuda, generator=g)
    pw = ops.pack_weight(w, b)
    ref = F.linear(rb(x), rb(w), b)
    v_ref = ref[:, 2 * D:].reshape(B, seq, D).permute(0, 2, 1)
    _multicast(lib, multicast)
    try:
        qk = torch.zeros(B * seq, 2 * D, dtype=torch.bfloat16, device=cuda)
        vt = torch.zeros(B * D, seq_pad, dtype=torch.bfloat16, device=cuda)
        d = ops.gemm(pw, [bf(x).contiguous()], qk, vt=vt, vt_col0=2 * D, vt_seq=seq, vt_seq_pad=seq_pad)
        torch.cuda.synchronize()
    finally:
        _multicast(lib, 1)
    check('qk part D %d' % D, qk, ref[:, :2 * D], 1e-2)
    check('v transposed D %d' % D, vt.reshape(B, D, seq_pad)[:, :, :seq], v_ref, 1e-2)
    assert (vt.reshape(B, D, seq_pad)[:, :, seq:] == 0).all()
    assert (d.block_n, d.n_tiles) == (bn, 9)
    assert d.m_tiles * d.n_tiles > 2 * 132


@pytest.mark.parametrize('k,Cin,Cout,bn', [(2, 72, 32, 32), (2, 64, 128, 128), (4, 96, 192, 192), (2, 600, 80, 96)])
def test_conv_transpose_block_n(cuda, k, Cin, Cout, bn):
    lib, ops = _lib_ops()
    g = torch.Generator(device='cuda').manual_seed(k + Cin + Cout)
    NB, H, W = 2, 23, 31
    x = torch.randn(NB, Cin, H, W, device=cuda, generator=g)
    w = torch.randn(Cin, Cout, k, k, device=cuda, generator=g) / Cin ** 0.5
    b = torch.randn(Cout, device=cuda, generator=g)
    pw = ops.pack_weight_convT(w, b, k)
    src = to_nhwc(x).reshape(NB * H * W, -1)
    out = torch.full((NB, H * k, W * k, ops.pad_to(Cout, 8) + 8), SENTINEL, dtype=torch.bfloat16, device=cuda)
    d = ops.gemm_convT(pw, src, (NB, H, W), out)
    ref = F.conv_transpose2d(rb(x), rb(w), b, stride=k)
    check('convT k%d %d->%d' % (k, Cin, Cout), from_nhwc(out, Cout), ref, 1e-2)
    assert (out[..., Cout:] == SENTINEL).all()
    assert d.block_n == bn


@pytest.mark.parametrize('N,n2', [(192, 16), (256, 4), (96, 1)])
def test_fused_tail_block_n(cuda, N, n2):
    """fused trailing layer over a whole 96-, 192- or 256-column row (1x1 conv): the half-row partial sums of lanes
    l and l ^ 16 meet in a warp shuffle"""
    lib, ops = _lib_ops()
    g = torch.Generator(device='cuda').manual_seed(N + n2)
    NB, H, W, cs = 2, 30, 41, [32, 136]
    xs = [torch.randn(NB, c, H, W, device=cuda, generator=g) for c in cs]
    w = torch.randn(N, sum(cs), 1, 1, device=cuda, generator=g) / sum(cs) ** 0.5
    b = torch.randn(N, device=cuda, generator=g)
    w2 = torch.randn(n2, N, device=cuda, generator=g) / N ** 0.5
    b2 = torch.randn(n2, device=cuda, generator=g)
    pw = ops.pack_weight(w, b, src_c=cs)
    outs, tails = [], []
    for _ in range(2):
        out = torch.full((NB, H, W, N), SENTINEL, dtype=torch.bfloat16, device=cuda)
        out3 = torch.zeros(NB, H, W, 16, dtype=torch.float32, device=cuda)
        d = ops.gemm(pw, [to_nhwc(x) for x in xs], out, image=(NB, H, W), act=ops.ACT_RELU,
                     tail=(w2, b2, ops.ACT_SOFTPLUS), tail_out=out3)
        outs.append(out)
        tails.append(out3)
    torch.cuda.synchronize()
    mid = F.relu(F.conv2d(torch.cat([rb(x) for x in xs], 1), rb(w), b))
    ref = F.softplus(F.conv2d(mid, w2.view(n2, N, 1, 1), b2))
    check('tail %d->%d' % (N, n2), tails[0][..., :n2].permute(0, 3, 1, 2), ref, 2e-3)
    check('tail main %d' % N, from_nhwc(outs[0], N), mid, 1e-2)
    assert torch.equal(tails[0], tails[1]) and torch.equal(outs[0], outs[1])
    assert (d.block_n, d.n_tiles) == (N, 1)


@pytest.mark.parametrize('tile', [(8, 16), (4, 32), (16, 8), (1, 128), (32, 4)])
@pytest.mark.parametrize('N', [256, 544])
def test_conv1x1_tiles(cuda, tile, N):
    """1x1 conv (a_mode 1) through the 4-D bf16 bulk-store epilogue at every pixel-tile shape"""
    lib, ops = _lib_ops()
    g = torch.Generator(device='cuda').manual_seed(N + tile[0])
    NB, H, W, Cin = 2, 37, 45, 200
    x = torch.randn(NB, Cin, H, W, device=cuda, generator=g)
    w = torch.randn(N, Cin, 1, 1, device=cuda, generator=g) / Cin ** 0.5
    b = torch.randn(N, device=cuda, generator=g)
    pw = ops.pack_weight(w, b)
    out = torch.full((NB, H, W, N + 16), SENTINEL, dtype=torch.bfloat16, device=cuda)
    d = ops.gemm(pw, [to_nhwc(x)], out, image=(NB, H, W), act=ops.ACT_RELU, tile=tile)
    ref = F.relu(F.conv2d(rb(x), rb(w), b))
    check('conv1x1 -> %d tile %s' % (N, tile), from_nhwc(out, N), ref, 1e-2)
    assert (out[..., N:] == SENTINEL).all()
    assert (d.bh, d.bw) == tile and d.block_n in (128, 192, 256)


@pytest.mark.parametrize('tile', [(8, 16), (4, 32)])
@pytest.mark.parametrize('cs,N,bn', [([40, 72], 96, 96), ([256], 256, 128), ([64, 32], 192, 192)])
def test_conv3x3_pinned_tile(cuda, tile, cs, N, bn):
    """3x3 conv through pf_gemm_kernel (pinned pixel tile: one TMA box per tap), partial last channel chunks"""
    lib, ops = _lib_ops()
    g = torch.Generator(device='cuda').manual_seed(N + sum(cs))
    NB, H, W = 2, 29, 47
    xs = [torch.randn(NB, c, H, W, device=cuda, generator=g) for c in cs]
    w = torch.randn(N, sum(cs), 3, 3, device=cuda, generator=g) / (9 * sum(cs)) ** 0.5
    b = torch.randn(N, device=cuda, generator=g)
    pw = ops.pack_weight(w, b, src_c=cs)
    out = torch.full((NB, H, W, N + 8), SENTINEL, dtype=torch.bfloat16, device=cuda)
    d = ops.gemm(pw, [to_nhwc(x) for x in xs], out, image=(NB, H, W), tile=tile)
    ref = F.conv2d(torch.cat([rb(x) for x in xs], 1), rb(w), b, padding=1)
    check('conv3x3 %s -> %d tile %s' % (cs, N, tile), from_nhwc(out, N), ref, 1e-2)
    assert (out[..., N:] == SENTINEL).all()
    assert (d.bh, d.bw) == tile and d.block_n == bn
