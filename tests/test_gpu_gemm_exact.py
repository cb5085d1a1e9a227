"""Bit-exact integer probes of pf_gemm_kernel and pf_conv3_halo_kernel (tests/exact_ref.py).

Every operand is a small integer (weights in {-1, 0, 1}, powers of two for gamma and the BN-fold scale), so every
partial sum is exact in fp32 and the kernel output must EQUAL the fp64 reference rounded once to the output dtype.  A
lost, doubled or misplaced product term anywhere (a channel of a partial 64-channel chunk, a tap at a tile edge, a k16
step of a zero-padded chunk, a halo row from the next image) is a mismatch, and the assertion message names its m-tile,
n-tile and pixel tile.  Each case also checks that columns beyond N keep their sentinel and that two launches give the
same bits.  The out-of-bounds cases put NaN wherever the kernels must not read (pad channels, rows past M, the image
after the last) and require the result to stay bit-identical to the clean run.
"""
import zlib

import pytest
import torch
import torch.nn.functional as F

import exact_ref as er
from exact_ref import Layout, assert_exact
from test_gpu_gemm_tiles import WIDTH_CASES

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

SENTINEL = 3.0
NAN = float('nan')


def _lib_ops():
    from patchfusion_b200 import lib, ops
    return lib, ops


def _gen(*key):
    return torch.Generator(device='cuda').manual_seed(zlib.crc32(repr(key).encode()))


def _bits(t):
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _same_bits(a, b):
    return torch.equal(_bits(a), _bits(b))


def _nhwc(x, ld=None, fill=0.0, nb=None):
    """fp32 NCHW integers -> bf16 NHWC [nb or NB, H, W, ld]; channels [C, pad8(C)) are 0, [pad8(C), ld) and images
    past NB hold `fill`"""
    from patchfusion_b200 import ops
    B, C, H, W = x.shape
    c8 = ops.pad_to(C, 8)
    ld = c8 if ld is None else ld
    out = torch.full((nb or B, H, W, ld), fill, dtype=torch.bfloat16, device=x.device)
    out[:B, :, :, :c8] = 0
    out[:B, :, :, :C] = x.permute(0, 2, 3, 1).to(torch.bfloat16)
    return out


def _want_nhwc(ref64, dtype=torch.bfloat16):
    return er.round_to(ref64, dtype).permute(0, 2, 3, 1)


class _Opt:
    """set a pf_set_option switch for the duration of a block, restoring the default"""

    def __init__(self, which, value, default=1):
        self.which, self.value, self.default = which, value, default

    def __enter__(self):
        lib, _ = _lib_ops()
        lib.call('pf_set_option', self.which, self.value)

    def __exit__(self, *a):
        lib, _ = _lib_ops()
        lib.call('pf_set_option', self.which, self.default)


def _twice(launch):
    """run launch() (-> desc, [outputs]) twice on fresh outputs; the two runs must agree bit for bit"""
    d, a = launch()
    _, b = launch()
    torch.cuda.synchronize()
    for i, (x, y) in enumerate(zip(a, b)):
        assert _same_bits(x, y), 'output %d: two identical launches differ' % i
    return d, a


def _skip_sm(bn):
    if torch.cuda.get_device_properties(0).multi_processor_count != 132 and bn in (128, 256):
        pytest.skip('the 128 / 256 choice depends on the SM count (132 on an H100 SXM)')


# ---------------------------------------------------------------------------------------------------- linear
def _linear_case(M, K, N, mode, multicast, g, out_col0=0, act=None, m_buf=None, a_ld=None, a_fill=0.0):
    """(launch, want, layout-col0, extra columns): a_mode 0 GEMM on integer probes.  mode: bf16 / f32 / gamma."""
    lib, ops = _lib_ops()
    x, amax = er.int_acts((M, K), g)
    w, wl1 = er.int_weights((N, K), g, er.density_for(K))
    b, bmax = er.int_bias(N, g)
    pw = ops.pack_weight(w, b)
    ld = a_ld or ops.pad_to(K, 8)
    xa = torch.full((m_buf or M, ld), a_fill, dtype=torch.bfloat16, device='cuda')
    xa[:M, :ops.pad_to(K, 8)] = 0
    xa[:M, :K] = x.to(torch.bfloat16)
    ref = er.ref_linear(x, w, b)
    act = act or ops.ACT_NONE
    if act == ops.ACT_RELU:
        ref = F.relu(ref)
    ocols = out_col0 + ops.pad_to(N, 8) + 8
    if mode == 'gamma':
        res, rmax = er.int_acts((M, ocols), g, amax=8)
        gam, gmax = er.pow2(N, g)
        er.check_bound(er.psum_bound(amax, wl1, bmax, scale=gmax, extra=rmax))
        want = res.double().clone()
        want[:, out_col0:out_col0 + N] += gam.double() * ref
        want = want.float()
    else:
        er.check_bound(er.psum_bound(amax, wl1, bmax))
        dt = torch.float32 if mode == 'f32' else torch.bfloat16
        want = torch.full((M, ocols), SENTINEL, dtype=dt, device='cuda')
        want[:, out_col0:out_col0 + N] = er.round_to(ref, dt)

    def launch():
        if mode == 'gamma':
            out = res.clone()
            d = ops.gemm(pw, [xa], out, gamma=gam, out_col0=out_col0, src_c=[K], M=M, act=act)
        else:
            out = torch.full((M, ocols), SENTINEL, dtype=want.dtype, device='cuda')
            d = ops.gemm(pw, [xa], out, act=act, out_col0=out_col0, src_c=[K], M=M)
        return d, [out]

    with _Opt(lib.OPT_GEMM_MULTICAST, multicast):
        d, (out,) = _twice(launch)
    return d, out, want, xa, launch


@pytest.mark.parametrize('M,N,bn,nt', WIDTH_CASES)
@pytest.mark.parametrize('mode', ['bf16', 'f32', 'gamma'])
@pytest.mark.parametrize('multicast', [0, 1])
def test_linear_exact_block_n(cuda, M, N, bn, nt, mode, multicast):
    """every compiled width, K = 592 (partial last chunk), the bf16 bulk store (bn % 64 == 0) or direct store, the fp32
    store and the fp32 gamma reduce-add; whole rows compared, so the sentinel columns beyond N are checked too"""
    _skip_sm(bn)
    d, out, want, _, _ = _linear_case(M, 592, N, mode, multicast, _gen('lin', M, N, mode))
    assert_exact('linear %dx592x%d %s mc %d' % (M, N, mode, multicast), out, want, Layout.from_desc(d))
    assert (d.block_n, d.n_tiles) == (bn, nt)


@pytest.mark.parametrize('M,K,N,mode,col0', [
    (300, 32, 96, 'bf16', 0),           # K < one chunk, 3 m-tiles (the last partial), block_n 96: direct store
    (300, 32, 256, 'f32', 8),           # fp32 direct store at column 8
    (1037, 1024, 384, 'bf16', 64),      # 16 chunks, bulk store at out_col0 64
    (9333, 32, 1024, 'gamma', 0),       # 73 m-tiles: odd count under multicast, one short K block
    (9333, 1024, 150, 'bf16', 16),      # block_n 32, five n-tiles with a narrow last one
    (777, 592, 200, 'gamma', 32),       # fp32 reduce-add into a wider residual stream at column 32
    (20000, 1024, 80, 'f32', 0),        # 157 m-tiles, block_n 96
    (8398, 592, 1001, 'bf16', 0),       # block_n 256, rows that end inside a 16-byte piece: nothing written past N
    (8398, 592, 1001, 'f32', 0),
    (8398, 592, 998, 'gamma', 0),
])
@pytest.mark.parametrize('multicast', [0, 1])
def test_linear_exact_shapes(cuda, M, K, N, mode, col0, multicast):
    _, ops = _lib_ops()
    d, out, want, _, _ = _linear_case(M, K, N, mode, multicast, _gen('lins', M, K, N), out_col0=col0,
                                      act=ops.ACT_RELU if mode == 'bf16' else None)
    assert_exact('linear %dx%dx%d %s col0 %d mc %d' % (M, K, N, mode, col0, multicast), out, want,
                 Layout.from_desc(d, col0=-col0))


@pytest.mark.parametrize('M,K,N,mode', [(1037, 200, 384, 'bf16'), (9333, 72, 1024, 'gamma'), (300, 40, 96, 'f32')])
def test_linear_oob_poison(cuda, M, K, N, mode):
    """NaN in source columns [pad8(K), ld) and in rows past M of a larger A buffer (passed with M=): the kernel must
    read neither, so the output is the clean run's, bit for bit"""
    g = ('linp', M, K, N)
    d, clean, want, _, _ = _linear_case(M, K, N, mode, 1, _gen(*g))
    _, ops = _lib_ops()
    _, dirty, _, xa, _ = _linear_case(M, K, N, mode, 1, _gen(*g), m_buf=M + 77, a_ld=ops.pad_to(K, 8) + 64, a_fill=NAN)
    assert torch.isnan(xa[M:]).all() and torch.isnan(xa[:M, ops.pad_to(K, 8):]).all()
    assert torch.isfinite(dirty).all()
    assert_exact('linear NaN-poisoned', dirty, clean, Layout.from_desc(d))
    assert_exact('linear clean', clean, want, Layout.from_desc(d))


@pytest.mark.parametrize('D,seq,bn', [(384, 1500, 128), (768, 1400, 256)])
@pytest.mark.parametrize('multicast', [0, 1])
def test_qkv_vt_exact(cuda, D, seq, bn, multicast):
    """fused qkv projection: q/k through the bulk store, V written transposed; V^T columns [seq, seq_pad) stay 0"""
    lib, ops = _lib_ops()
    if torch.cuda.get_device_properties(0).multi_processor_count != 132:
        pytest.skip('tile counts chosen for 132 SMs')
    g = _gen('qkv', D, seq)
    B, K = 4, 64
    seq_pad = ops.pad_to(seq, 8)
    x, amax = er.int_acts((B * seq, K), g)
    w, wl1 = er.int_weights((3 * D, K), g)
    b, bmax = er.int_bias(3 * D, g)
    er.check_bound(er.psum_bound(amax, wl1, bmax))
    pw = ops.pack_weight(w, b)
    ref = er.round_to(er.ref_linear(x, w, b), torch.bfloat16)
    xa = x.to(torch.bfloat16).contiguous()

    def launch():
        qk = torch.zeros(B * seq, 2 * D, dtype=torch.bfloat16, device=cuda)
        vt = torch.zeros(B * D, seq_pad, dtype=torch.bfloat16, device=cuda)
        d = ops.gemm(pw, [xa], qk, vt=vt, vt_col0=2 * D, vt_seq=seq, vt_seq_pad=seq_pad)
        return d, [qk, vt]

    with _Opt(lib.OPT_GEMM_MULTICAST, multicast):
        d, (qk, vt) = _twice(launch)
    assert_exact('qk D %d' % D, qk, ref[:, :2 * D], Layout.from_desc(d))
    v = vt.view(B, D, seq_pad)
    assert_exact('V^T D %d (token-major)' % D, v[:, :, :seq].permute(0, 2, 1).reshape(B * seq, D), ref[:, 2 * D:],
                 Layout.from_desc(d, col0=2 * D))
    assert (v[:, :, seq:] == 0).all() and not torch.signbit(v[:, :, seq:].float()).any()
    assert (d.block_n, d.n_tiles) == (bn, 9)


# ---------------------------------------------------------------------------------------------------- 1x1 conv
def _conv_case(NB, H, W, cs, N, g, k=1, tile=None, act=None, ld_extra=0, fill=0.0, nb_buf=None, resample_from=None,
               scale=None, out_col0=0, density=None, cluster=None):
    """a_mode 1 conv (k = 1 or 3) on integer probes; resample_from[i] = (h, w) reads source i through the fused
    bilinear resample.  Returns (desc, out, want, launch)."""
    lib, ops = _lib_ops()
    rs = resample_from or [None] * len(cs)
    xs, amax = [], 0.0
    for c, r in zip(cs, rs):
        h, w_ = r if r else (H, W)
        if r:
            er.dyadic_ratio(h, H)
            er.dyadic_ratio(w_, W)
        x, amax = er.int_acts((NB, c, h, w_), g)
        xs.append(x)
    K = k * k * sum(cs)
    wt, wl1 = er.int_weights((N, sum(cs), k, k), g, er.density_for(K) if density is None else density)
    b, bmax = er.int_bias(N, g)
    if scale is not None:
        s, smax = er.pow2(N, g)
        pw = ops.pack_weight(wt, None, src_c=cs, scale=s, shift=b)
        er.check_bound(er.psum_bound(amax, wl1, bmax, scale=smax))
        weff = wt * s.view(-1, 1, 1, 1)
    else:
        pw = ops.pack_weight(wt, b, src_c=cs)
        er.check_bound(er.psum_bound(amax, wl1, bmax))
        weff = wt
    srcs = [_nhwc(x, ops.pad_to(c, 8) + ld_extra, fill, nb_buf) for x, c in zip(xs, cs)]
    up = [er.ref_resize(x, (H, W)) if r else x.double() for x, r in zip(xs, rs)]
    ref = er.ref_conv(torch.cat(up, 1), weff, b, padding=k // 2)
    if act == ops.ACT_RELU:
        ref = F.relu(ref)
    ocols = out_col0 + ops.pad_to(N, 8) + 8
    want = torch.full((NB, H, W, ocols), SENTINEL, dtype=torch.bfloat16, device='cuda')
    want[..., out_col0:out_col0 + N] = _want_nhwc(ref)
    resample = [r is not None for r in rs] if any(rs) else None

    def launch():
        out = torch.full((NB, H, W, ocols), SENTINEL, dtype=torch.bfloat16, device='cuda')
        d = ops.gemm(pw, srcs, out, image=(NB, H, W), act=act or ops.ACT_NONE, tile=tile, resample=resample,
                     out_col0=out_col0)
        return d, [out]

    if cluster is None:
        d, (out,) = _twice(launch)
    else:
        with _Opt(lib.OPT_HALO_MULTICAST, cluster):
            d, (out,) = _twice(launch)
    return d, out, want, launch, srcs


@pytest.mark.parametrize('tile', [(8, 16), (4, 32), (16, 8), (1, 128), (32, 4)])
@pytest.mark.parametrize('N', [256, 544])
def test_conv1x1_exact_tiles(cuda, tile, N):
    """1x1 conv at every pixel-tile shape through the 4-D bulk store, 200 channels (a partial second chunk)"""
    _, ops = _lib_ops()
    d, out, want, _, _ = _conv_case(2, 37, 45, [200], N, _gen('c1', N, tile), tile=tile, act=ops.ACT_RELU)
    assert_exact('conv1x1 -> %d tile %s' % (N, tile), out, want, Layout.from_desc(d))
    assert (d.bh, d.bw) == tile


@pytest.mark.parametrize('N', [96, 192])
def test_conv1x1_exact_two_sources(cuda, N):
    d, out, want, _, _ = _conv_case(2, 30, 41, [32, 136], N, _gen('c1s', N))
    assert_exact('conv1x1 [32, 136] -> %d' % N, out, want, Layout.from_desc(d))


def test_conv1x1_exact_bn_fold(cuda):
    """BN fold: power-of-two scale packed into the weights, integer shift, output at channel offset 64"""
    d, out, want, _, _ = _conv_case(1, 20, 23, [96], 48, _gen('bn'), scale=True, out_col0=64)
    assert_exact('conv1x1 BN fold at col 64', out, want, Layout.from_desc(d, col0=-64))


# ---------------------------------------------------------------------------------------------------- 3x3 halo
HALO_TABLE = [([32, 256, 256], 544, 192, 3), ([64], 768, 192, 4), ([40, 64], 256, 128, 2), ([96], 56, 64, 1),
              ([8], 96, 32, 3), ([136], 32, 32, 1)]


@pytest.mark.parametrize('cs,N,bn,nt', HALO_TABLE)
@pytest.mark.parametrize('cluster', [0, 1, 2])
def test_halo_exact_block_n(cuda, cs, N, bn, nt, cluster):
    """5 x 50 x 70: 180 pixel tiles of 16 x 8, partial at the bottom (50 % 16) and right (70 % 8) of every image, so
    tiles sit on image boundaries; clusters of 1, 2 and 4 CTAs sharing the weights"""
    _, ops = _lib_ops()
    d, out, want, _, _ = _conv_case(5, 50, 70, cs, N, _gen('halo', N, len(cs)), k=3, act=ops.ACT_RELU, cluster=cluster)
    assert_exact('halo %s -> %d cl-opt %d' % (cs, N, cluster), out, want, Layout.from_desc(d))
    assert (d.block_n, d.n_tiles) == (bn, nt)


def test_halo_exact_residuals_and_relu_copy(cuda):
    _, ops = _lib_ops()
    g = _gen('res')
    NB, H, W, C = 3, 29, 37, 64
    x, amax = er.int_acts((NB, C, H, W), g)
    r1, _ = er.int_acts((NB, C, H, W), g)
    r2, _ = er.int_acts((NB, C, H, W), g)
    wt, wl1 = er.int_weights((C, C, 3, 3), g, er.density_for(9 * C))
    b, bmax = er.int_bias(C, g)
    er.check_bound(er.psum_bound(amax, wl1, bmax, extra=4))
    pw = ops.pack_weight(wt, b)
    ref = er.ref_conv(x, wt, b) + r1.double() + r2.double()
    src, n1, n2 = _nhwc(x), _nhwc(r1), _nhwc(r2)

    def launch():
        out = torch.zeros(NB, H, W, C, dtype=torch.bfloat16, device=cuda)
        out2 = torch.zeros_like(out)
        d = ops.gemm(pw, [src], out, image=(NB, H, W), res1=n1, res2=n2, out2=out2)
        return d, [out, out2]

    d, (out, out2) = _twice(launch)
    assert_exact('conv + res1 + res2', out, _want_nhwc(ref), Layout.from_desc(d))
    assert_exact('relu copy', out2, _want_nhwc(F.relu(ref)), Layout.from_desc(d))


@pytest.mark.parametrize('k,cs,N,n2,act2', [(3, [64], 192, 4, 'relu'), (3, [40, 64], 128, 16, 'none'),
                                            (1, [32, 136], 256, 4, 'relu'), (1, [32, 136], 192, 16, 'none'),
                                            (1, [128], 96, 1, 'relu')])
def test_fused_tail_exact(cuda, k, cs, N, n2, act2):
    """fused trailing 1x1 layer (halo kernel for k = 3, pf_gemm_kernel for k = 1): |main| <= 256 by construction, so
    the tail is exact whether it reads the fp32 accumulator or the bf16 store"""
    _, ops = _lib_ops()
    g = _gen('tail', k, N, n2)
    NB, H, W = 2, 30, 41
    xs = [er.int_acts((NB, c, H, W), g)[0] for c in cs]
    wt, wl1 = er.int_weights((N, sum(cs), k, k), g, 0.2, l1max=120)
    b, bmax = er.int_bias(N, g)
    assert 2 * wl1 + bmax <= 256
    w2, w2l1 = er.int_weights((n2, N), g)
    b2, _ = er.int_bias(n2, g)
    er.check_bound(er.psum_bound(256, w2l1, 8))
    pw = ops.pack_weight(wt, b, src_c=cs)
    A = dict(relu=ops.ACT_RELU, none=ops.ACT_NONE)
    mid = F.relu(er.ref_conv(torch.cat(xs, 1), wt, b, padding=k // 2))
    t = F.conv2d(mid, w2.double().view(n2, N, 1, 1), b2.double())
    t = F.relu(t) if act2 == 'relu' else t
    srcs = [_nhwc(x) for x in xs]

    def launch():
        out = torch.full((NB, H, W, N), SENTINEL, dtype=torch.bfloat16, device=cuda)
        out3 = torch.full((NB, H, W, 16), SENTINEL, dtype=torch.float32, device=cuda)
        d = ops.gemm(pw, srcs, out, image=(NB, H, W), act=ops.ACT_RELU, tail=(w2, b2, A[act2]), tail_out=out3)
        return d, [out, out3]

    d, (out, out3) = _twice(launch)
    assert d.n_tiles == 1
    assert_exact('tail main', out, _want_nhwc(mid), Layout.from_desc(d))
    want3 = torch.full_like(out3, SENTINEL)
    want3[..., :n2] = _want_nhwc(t, torch.float32)
    assert_exact('tail %d -> %d %s' % (N, n2, act2), out3, want3, Layout('nhwc', 16, d.bh, d.bw))


# ---------------------------------------------------------------------------------------------------- resample
@pytest.mark.parametrize('NB,H,W,srcs,N,cluster', [
    (3, 25, 37, [(13, 19, 64)], 64, 1),                                   # x2 (ratio 1/2)
    (3, 25, 37, [(7, 10, 72), (25, 37, 40), (13, 19, 136)], 96, 1),       # 1/4, direct, 1/2; partial chunks
    (3, 33, 49, [(25, 37, 136)], 544, 1),                                 # ratio 3/4
    (7, 49, 73, [(25, 37, 64), (49, 73, 32)], 192, 0),                    # >= 132 tiles: clusters of 1, 2 and 4
    (7, 49, 73, [(25, 37, 64), (49, 73, 32)], 192, 1),
    (7, 49, 73, [(25, 37, 64), (49, 73, 32)], 192, 2),
])
def test_halo_exact_fused_resample(cuda, NB, H, W, srcs, N, cluster):
    """fused bilinear (align_corners) resample at dyadic ratios: the resampled bf16 values are exact"""
    _, ops = _lib_ops()
    cs = [c for _, _, c in srcs]
    rf = [(h, w) if (h, w) != (H, W) else None for h, w, _ in srcs]
    d, out, want, _, _ = _conv_case(NB, H, W, cs, N, _gen('rs', H, N, len(cs)), k=3, act=ops.ACT_RELU,
                                    resample_from=rf, cluster=cluster)
    assert_exact('halo resample %s -> %d @%dx%d cl-opt %d' % (srcs, N, H, W, cluster), out, want, Layout.from_desc(d))


@pytest.mark.parametrize('h,w,OH,OW,C', [(7, 10, 25, 37, 72), (13, 19, 25, 37, 128), (33, 49, 65, 97, 72),
                                         (33, 49, 65, 97, 128), (25, 37, 33, 49, 64)])
@pytest.mark.parametrize('separable', [0, 1])
def test_resize_bilinear_exact(cuda, h, w, OH, OW, C, separable):
    """pf_resize_bilinear at dyadic ratios: the direct kernel (C % 64 != 0 or < 4096 output pixels) and the tiled one
    (65 x 97 x 128), whose separable form is an option"""
    lib, ops = _lib_ops()
    er.dyadic_ratio(h, OH)
    er.dyadic_ratio(w, OW)
    g = _gen('rsz', h, OH, C)
    NB = 2
    x, _ = er.int_acts((NB, C, h, w), g)
    src = _nhwc(x, C + 16, NAN)
    want = torch.full((NB, OH, OW, C + 24), SENTINEL, dtype=torch.bfloat16, device=cuda)
    want[..., 8:8 + C] = _want_nhwc(er.ref_resize(x, (OH, OW)))
    outs = []
    with _Opt(lib.OPT_RESIZE_SEPARABLE, separable, default=0):
        for _ in range(2):
            out = torch.full_like(want, SENTINEL)
            ops.resize_bilinear(src, C, OH, OW, out, out_col0=8)
            outs.append(out)
        torch.cuda.synchronize()
    assert _same_bits(outs[0], outs[1])
    assert_exact('resize %dx%d -> %dx%d C %d' % (h, w, OH, OW, C), outs[0], want, Layout('nhwc', 64, 8, 32, col0=-8))


# ---------------------------------------------------------------------------------------------------- pinned tile, convT
@pytest.mark.parametrize('tile', [(8, 16), (4, 32)])
@pytest.mark.parametrize('cs,N,bn', [([40, 72], 96, 96), ([256], 256, 128), ([64, 32], 192, 192)])
def test_conv3x3_pinned_tile_exact(cuda, tile, cs, N, bn):
    """3x3 conv through pf_gemm_kernel with one TMA box per tap (pinned pixel tile), partial last channel chunks"""
    d, out, want, _, _ = _conv_case(2, 29, 47, cs, N, _gen('pin', N, tile), k=3, tile=tile)
    assert_exact('pinned %s -> %d tile %s' % (cs, N, tile), out, want, Layout.from_desc(d))
    assert (d.bh, d.bw) == tile and d.block_n == bn


def _convT_rows(t, k, cpad):
    """NHWC [NB, H k, W k, C] -> the GEMM's [NB H W, k k cpad] rows (input pixel, (tap, channel))"""
    NB, Hk, Wk, C = t.shape
    r = t.reshape(NB, Hk // k, k, Wk // k, k, C).permute(0, 1, 3, 2, 4, 5).reshape(-1, k * k, C)
    out = torch.zeros(r.shape[0], k * k, cpad, dtype=t.dtype, device=t.device)
    out[..., :C] = r
    return out.reshape(r.shape[0], -1)


@pytest.mark.parametrize('k,Cin,Cout,bn', [(2, 72, 32, 32), (2, 64, 128, 128), (4, 96, 192, 192), (2, 600, 80, 96)])
def test_conv_transpose_exact(cuda, k, Cin, Cout, bn):
    _, ops = _lib_ops()
    g = _gen('convT', k, Cin, Cout)
    NB, H, W = 2, 23, 31
    x, amax = er.int_acts((NB, Cin, H, W), g)
    w, wl1 = er.int_weights_convT((Cin, Cout, k, k), g, er.density_for(Cin))
    b, bmax = er.int_bias(Cout, g)
    er.check_bound(er.psum_bound(amax, wl1, bmax))
    pw = ops.pack_weight_convT(w, b, k)
    src = _nhwc(x).reshape(NB * H * W, -1)

    def launch():
        out = torch.full((NB, H * k, W * k, ops.pad_to(Cout, 8) + 8), SENTINEL, dtype=torch.bfloat16, device=cuda)
        return ops.gemm_convT(pw, src, (NB, H, W), out), [out]

    d, (out,) = _twice(launch)
    want = torch.full_like(out, SENTINEL)
    want[..., :Cout] = _want_nhwc(er.ref_conv_transpose(x, w, b, k))
    cpad = ops.pad_to(Cout, 32)
    assert_exact('convT k%d %d->%d' % (k, Cin, Cout), _convT_rows(out[..., :Cout], k, cpad),
                 _convT_rows(want[..., :Cout], k, cpad), Layout.from_desc(d))
    assert (out[..., Cout:] == SENTINEL).all()
    assert d.block_n == bn


# ---------------------------------------------------------------------------------------------------- tap shifts
@pytest.mark.parametrize('tap', range(9))
@pytest.mark.parametrize('tile', [None, (8, 16)])
def test_tap_shift(cuda, tap, tile):
    """w[n, c, ky, kx] = 1 iff n == c and 3 ky + kx == tap: the output is the input shifted by (ky - 1, kx - 1), zeros
    outside each image.  NB = 3 at 21 x 13: partial tiles at the bottom and right of every image for both the halo
    kernel (16 x 8) and the pinned-tile kernel (8 x 16); 72 channels, a partial second chunk."""
    _, ops = _lib_ops()
    g = _gen('tap', tap)
    NB, H, W, C = 3, 21, 13, 72
    x, _ = er.int_acts((NB, C, H, W), g, amax=100)
    wt = torch.zeros(C, C, 3, 3, device=cuda)
    ky, kx = divmod(tap, 3)
    ar = torch.arange(C, device=cuda)
    wt[ar, ar, ky, kx] = 1.0
    pw = ops.pack_weight(wt, None)
    want = F.pad(x, (1, 1, 1, 1))[:, :, ky:ky + H, kx:kx + W]
    src = _nhwc(x, fill=NAN, nb=NB + 1, ld=C + 8)
    out = torch.zeros(NB, H, W, C, dtype=torch.bfloat16, device=cuda)
    d = ops.gemm(pw, [src], out, image=(NB, H, W), tile=tile)
    torch.cuda.synchronize()
    assert_exact('tap %d shift (%d, %d) %s' % (tap, ky - 1, kx - 1, 'halo' if tile is None else 'pinned'),
                 out, _want_nhwc(want), Layout.from_desc(d))


# ---------------------------------------------------------------------------------------------------- OOB poisoning
@pytest.mark.parametrize('kind', ['conv1x1', 'halo', 'halo-mc', 'pinned', 'resample'])
def test_conv_oob_poison(cuda, kind):
    """NaN in source channels [pad8(C), ld) and in an extra image after the last one (source [NB + 1, H, W, ld],
    image = (NB, H, W)): the output must stay finite and equal to the clean run bit for bit"""
    _, ops = _lib_ops()
    NB, H, W = (7, 49, 73) if kind == 'halo-mc' else (3, 25, 37)
    k = 1 if kind == 'conv1x1' else 3
    cs = [36, 130]
    rf = [(13, 19), None] if kind == 'resample' else None
    kw = dict(k=k, tile=(8, 16) if kind == 'pinned' else None, act=ops.ACT_RELU, resample_from=rf)
    N = 96
    d, clean, want, _, _ = _conv_case(NB, H, W, cs, N, _gen('poison', kind), **kw)
    _, dirty, _, _, srcs = _conv_case(NB, H, W, cs, N, _gen('poison', kind), ld_extra=40, fill=NAN, nb_buf=NB + 1, **kw)
    assert all(torch.isnan(s[NB]).all() and torch.isnan(s[:NB, ..., ops.pad_to(c, 8):]).all() for s, c in zip(srcs, cs))
    assert torch.isfinite(dirty.float()).all()
    assert_exact('%s NaN-poisoned' % kind, dirty, clean, Layout.from_desc(d))
    assert_exact('%s clean' % kind, clean, want, Layout.from_desc(d))
    if kind == 'halo-mc':
        assert d.m_tiles * d.n_tiles >= torch.cuda.get_device_properties(0).multi_processor_count
