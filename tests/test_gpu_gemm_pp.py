"""pf_gemm_pp_kernel (whole 128 x 128 tiles per consumer warpgroup, ping-pong mainloops) on bit-exact integer probes
(tests/exact_ref.py).

Plain linear layers whose N is a multiple of 128 go through it: bias with no activation / ReLU through the bf16 bulk
store, the fp32 store, the fp32 gamma reduce-add, and a fused qkv projection with its V^T third stored from the
fragment.  Shapes cover a single row, m-tile edges, an odd m-tile count under multicast, CTAs where the second
warpgroup gets no tile, and N of one to 32 tiles.  GELU is not exact on integers: it is compared bit for bit with
pf_gemm_kernel's row-per-thread epilogue (the same fp32 operations in the same order).  Every case checks which kernel
ran.
"""
import pytest
import torch

import exact_ref as er
from exact_ref import Layout, assert_exact
from test_gpu_gemm_exact import NAN, _gen, _linear_case, _Opt, _same_bits

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(600)]

MS = [1, 127, 128, 129, 1037, 9333]
NS = [128, 1024, 3072, 4096]


def _lib_ops():
    from patchfusion_b200 import lib, ops
    return lib, ops


def _kernels(launch):
    """names of the kernels launch() runs"""
    lib, _ = _lib_ops()
    prof = lib.Profiler()
    torch.cuda.synchronize()
    prof.start()
    launch()
    torch.cuda.synchronize()
    return {r[0] for r in prof.stop()}


def _assert_pp(launch, multicast):
    lib, _ = _lib_ops()
    with _Opt(lib.OPT_GEMM_MULTICAST, multicast):
        names = _kernels(launch)
    assert names == {'pf_gemm_pp_kernel'}, names


@pytest.mark.parametrize('M', MS)
@pytest.mark.parametrize('N', NS)
@pytest.mark.parametrize('multicast', [0, 1])
def test_pp_linear_bias_exact(cuda, M, N, multicast):
    """bias, bf16 bulk store; whole rows compared, so the sentinel columns past N are checked too"""
    d, out, want, _, launch = _linear_case(M, 592, N, 'bf16', multicast, _gen('pp', M, N))
    assert_exact('pp linear %dx592x%d mc %d' % (M, N, multicast), out, want, Layout.from_desc(d))
    _assert_pp(launch, multicast)


@pytest.mark.parametrize('M', MS)
@pytest.mark.parametrize('mode', ['f32', 'gamma', 'relu'])
@pytest.mark.parametrize('multicast', [0, 1])
def test_pp_linear_epilogues_exact(cuda, M, mode, multicast):
    """fp32 store, fp32 gamma reduce-add into the residual stream, bias + ReLU (K = 1024: 16 whole K blocks)"""
    _, ops = _lib_ops()
    N = 1024
    d, out, want, _, launch = _linear_case(M, 1024, N, 'bf16' if mode == 'relu' else mode, multicast,
                                           _gen('ppe', M, mode), act=ops.ACT_RELU if mode == 'relu' else None)
    assert_exact('pp linear %dx1024x%d %s mc %d' % (M, N, mode, multicast), out, want, Layout.from_desc(d))
    _assert_pp(launch, multicast)


@pytest.mark.parametrize('M,N', [(1, 128), (129, 1024), (1037, 4096), (9333, 4096)])
@pytest.mark.parametrize('multicast', [0, 1])
def test_pp_gelu_matches_row_epilogue(cuda, M, N, multicast):
    """bias + exact-erf GELU: the same bits as pf_gemm_kernel's row-per-thread epilogue (bulk stores switched off)"""
    lib, ops = _lib_ops()
    g = torch.Generator(device='cuda').manual_seed(M * 7 + N)
    K = 1024
    x = (torch.randn(M, K, device='cuda', generator=g)).to(torch.bfloat16)
    w = torch.randn(N, K, device='cuda', generator=g) / K ** 0.5
    pw = ops.pack_weight(w, torch.randn(N, device='cuda', generator=g))

    def launch():
        out = torch.full((M, N), 3.0, dtype=torch.bfloat16, device='cuda')
        ops.gemm(pw, [x], out, act=ops.ACT_GELU)
        return out

    with _Opt(lib.OPT_GEMM_MULTICAST, multicast):
        got = launch()
        names = _kernels(launch)
        with _Opt(lib.OPT_TMA_EPILOGUE, 0):
            ref = launch()
            ref_names = _kernels(launch)
    torch.cuda.synchronize()
    assert names == {'pf_gemm_pp_kernel'} and ref_names == {'pf_gemm_kernel'}, (names, ref_names)
    assert _same_bits(got, ref), 'GELU: %d elements differ' % int((got != ref).sum())


@pytest.mark.parametrize('M,K,N,mode', [(1037, 200, 1024, 'bf16'), (9333, 72, 1024, 'gamma'), (300, 40, 128, 'f32')])
def test_pp_linear_oob_poison(cuda, M, K, N, mode):
    """NaN in source columns [pad8(K), ld) and in rows past M of a larger A buffer: the output is the clean run's"""
    _, ops = _lib_ops()
    key = ('ppp', M, K, N)
    d, clean, want, _, launch = _linear_case(M, K, N, mode, 1, _gen(*key))
    _, dirty, _, xa, _ = _linear_case(M, K, N, mode, 1, _gen(*key), m_buf=M + 77, a_ld=ops.pad_to(K, 8) + 64,
                                      a_fill=NAN)
    assert torch.isnan(xa[M:]).all() and torch.isnan(xa[:M, ops.pad_to(K, 8):]).all()
    assert torch.isfinite(dirty).all()
    assert_exact('pp linear NaN-poisoned', dirty, clean, Layout.from_desc(d))
    assert_exact('pp linear clean', clean, want, Layout.from_desc(d))
    _assert_pp(launch, 1)


@pytest.mark.parametrize('B,seq,D', [(9, 1037, 1024), (1, 1037, 1024), (3, 300, 384), (2, 100, 128)])
@pytest.mark.parametrize('multicast', [0, 1])
def test_pp_qkv_vt_exact(cuda, B, seq, D, multicast):
    """fused qkv projection: q / k through the bulk store, V^T from the fragment; images of odd length, so 8-token row
    groups and 128-row tiles straddle image boundaries; V^T columns [seq, seq_pad) stay 0"""
    lib, ops = _lib_ops()
    g = _gen('ppqkv', B, seq, D)
    K = 64
    seq_pad = ops.pad_to(seq, 64)
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
        return d, qk, vt

    with _Opt(lib.OPT_GEMM_MULTICAST, multicast):
        d, qk, vt = launch()
        _, qk2, vt2 = launch()
    torch.cuda.synchronize()
    assert _same_bits(qk, qk2) and _same_bits(vt, vt2), 'two identical launches differ'
    assert_exact('pp qk B %d seq %d D %d' % (B, seq, D), qk, ref[:, :2 * D], Layout.from_desc(d))
    v = vt.view(B, D, seq_pad)
    assert_exact('pp V^T B %d seq %d D %d (token-major)' % (B, seq, D),
                 v[:, :, :seq].permute(0, 2, 1).reshape(B * seq, D), ref[:, 2 * D:], Layout.from_desc(d, col0=2 * D))
    assert (v[:, :, seq:] == 0).all() and not torch.signbit(v[:, :, seq:].float()).any()
    _assert_pp(lambda: launch(), multicast)
