"""fp64 sweep of the GEMM / conv epilogue activations (ReLU, GELU, softplus) over every bf16 input in a range.

Setup: A[m, 0] = x_m, W[n, 0] = 1 and every other weight 0, so the accumulator is exactly x_m; the bias b_n is an fp32
offset in [-0.5, 0.5] with full mantissa bits.  The kernel's `acc + bias` is then the same single fp32 rounding as
torch's z = x.float()[:, None] + b, and the reference is act(z) in fp64.  x_m runs over every bf16 value with |x| in
[2^-8, 24], both signs, and 0 (3203 rows), which also crosses softplus's z > 20 switch.

Paths: a full n-tile (N = 256: bulk-store epilogue, `gelu_erf2`) and a partial last n-tile (N = 200, block_n 32: the
direct-store epilogue, `gelu_erf2` on full 16-column chunks and the scalar `gelu_erf` on the partial one); the fp32
output through the bulk store (linear) and through the direct store (1x1 conv); the halo-kernel epilogue (3x3 conv,
centre tap of channel 0); the fused trailing layer's act2 (scalar `gelu_erf`, fp32 out3) with a one-hot w2.

Bounds, fixed in advance from documented errors (eps = error of the fp32 value the kernel computes before its store):
- GELU: erf by Abramowitz-Stegun 7.1.26 has |error| <= 1.5e-7, i.e. 1.5e-7 |z| / 2 in 0.5 z (1 + erf); the fp32
  evaluation (MUFU reciprocal and exp2, the cancellation in 1 - p t exp(-u^2) and in 0.5 z + 0.5 |z| erf) adds a few
  2^-24 |z|: eps = |z| (0.75e-7 + 4 * 2^-24).
- softplus: expf and log1pf within 2 ulp each, and the error of exp passes through log1p damped by sigmoid(z) <=
  softplus(z): eps = 8 * 2^-24 |softplus(z)|.  The z > 20 switch returns z, 2e-9 below softplus(20).
- both: an absolute floor of 2^-126 for results below the fp32 normal range (exp2.approx flushes them).
- bf16 outputs: |got - ref| <= 2^-8 (|ref| + eps) + eps, i.e. half a bf16 ulp of the fp32 value plus eps.
- fp32 outputs: |got - ref| <= eps + 2^-23 |ref| (two fp32 roundings).
- ReLU: exact, compared bit for bit.
GELU at z <~ -4 is tiny and has a large relative error; the bound there is absolute by design.
"""
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]

FLOOR = 2.0 ** -126
U = 2.0 ** -24


def _lib_ops():
    from patchfusion_b200 import lib, ops
    return lib, ops


def _xs(dev):
    """every bf16 value with |x| in [2^-8, 24], both signs, and 0"""
    lo = torch.tensor(2.0 ** -8, dtype=torch.bfloat16).view(torch.int16).item()
    hi = torch.tensor(24.0, dtype=torch.bfloat16).view(torch.int16).item()
    pos = torch.arange(lo, hi + 1, dtype=torch.int16).view(torch.bfloat16)
    return torch.cat([-pos.flip(0), torch.zeros(1, dtype=torch.bfloat16), pos]).to(dev)


def _bias(n, seed, dev):
    b = torch.rand(n, generator=torch.Generator().manual_seed(seed), dtype=torch.float32) - 0.5
    return b.to(dev)


def _ref(act, z):
    z = z.double()
    if act == 'relu':
        return z.clamp_min(0)
    if act == 'gelu':
        return 0.5 * z * (1.0 + torch.erf(z / 2.0 ** 0.5))
    return torch.log1p(torch.exp(z))


def _eps(act, z, ref):
    if act == 'gelu':
        return z.double().abs() * (0.75e-7 + 4 * U) + FLOOR
    return 8 * U * ref.abs() + FLOOR


def _check(name, act, got, z):
    """got: kernel output, z: the fp32 pre-activation (same shape)"""
    ref = _ref(act, z)
    if act == 'relu':
        want = ref.to(got.dtype)
        bad = (got.double() != want.double()) | torch.isnan(got.double())
        assert not bad.any(), '%s: %d ReLU outputs differ, first at z = %r' % (name, int(bad.sum()), z[bad][0].item())
        print('%-44s exact' % name)
        return
    eps = _eps(act, z, ref)
    if got.dtype == torch.bfloat16:
        bound = 2.0 ** -8 * (ref.abs() + eps) + eps
    else:
        bound = eps + 2.0 ** -23 * ref.abs()
    err = (got.double() - ref).abs()
    ratio = err / bound
    i = int(torch.argmax(torch.nan_to_num(ratio, nan=float('inf'))).item())
    worst = ratio.flatten()[i].item()
    zi, gi, ri = z.flatten()[i].item(), got.double().flatten()[i].item(), ref.flatten()[i].item()
    print('%-44s worst |err| / bound = %.3f at z = %.9g (got %.9g, fp64 %.9g, |err| %.3g)' % (name, worst, zi, gi, ri,
                                                                                            abs(gi - ri)))
    assert torch.isfinite(got.double()).all(), '%s: non-finite output' % name
    assert worst <= 1.0, '%s: error %.3g > bound %.3g at z = %.9g (got %.9g, fp64 %.9g)' % (
        name, abs(gi - ri), bound.flatten()[i].item(), zi, gi, ri)


ACTS = ['relu', 'gelu', 'softplus']


def _acts(ops):
    return dict(relu=ops.ACT_RELU, gelu=ops.ACT_GELU, softplus=ops.ACT_SOFTPLUS)


def _linear(ops, x, N, bias, act, out_dtype):
    M = x.shape[0]
    w = torch.zeros(N, 8, device=x.device)
    w[:, 0] = 1.0
    pw = ops.pack_weight(w, bias)
    xa = torch.zeros(M, 8, dtype=torch.bfloat16, device=x.device)
    xa[:, 0] = x
    out = torch.full((M, N), 7.0, dtype=out_dtype, device=x.device)
    d = ops.gemm(pw, [xa], out, act=_acts(ops)[act])
    torch.cuda.synchronize()
    return d, out


@pytest.mark.parametrize('act', ACTS)
@pytest.mark.parametrize('N,bn', [(256, 128), (200, 32)])
@pytest.mark.parametrize('out_dtype', ['bf16', 'f32'])
def test_linear_epilogue_act(cuda, act, N, bn, out_dtype):
    """bf16: N = 256 takes the bulk store (gelu_erf2), N = 200 the direct store with a partial last chunk (gelu_erf2 and
    gelu_erf); fp32: the fp32 bulk store"""
    _, ops = _lib_ops()
    x = _xs(cuda)
    b = _bias(N, N, cuda)
    dt = torch.bfloat16 if out_dtype == 'bf16' else torch.float32
    d, out = _linear(ops, x, N, b, act, dt)
    z = x.float()[:, None] + b[None, :]
    _check('linear N %d %s -> %s' % (N, act, out_dtype), act, out, z)
    assert d.block_n == bn


@pytest.mark.parametrize('act', ACTS)
@pytest.mark.parametrize('N', [256, 200])
def test_conv1x1_fp32_direct_store_act(cuda, act, N):
    """1x1 conv with an fp32 output: the direct-store epilogue (per-element predicated chunk at N = 200)"""
    _, ops = _lib_ops()
    x = _xs(cuda)
    M = x.shape[0]
    b = _bias(N, N + 1, cuda)
    w = torch.zeros(N, 8, 1, 1, device=cuda)
    w[:, 0] = 1.0
    pw = ops.pack_weight(w, b)
    src = torch.zeros(1, 1, M, 8, dtype=torch.bfloat16, device=cuda)
    src[0, 0, :, 0] = x
    out = torch.full((1, 1, M, N), 7.0, dtype=torch.float32, device=cuda)
    ops.gemm(pw, [src], out, image=(1, 1, M), act=_acts(ops)[act])
    torch.cuda.synchronize()
    _check('conv1x1 N %d %s -> f32 direct' % (N, act), act, out[0, 0], x.float()[:, None] + b[None, :])


@pytest.mark.parametrize('act', ACTS)
@pytest.mark.parametrize('N', [256, 200])
def test_halo_epilogue_act(cuda, act, N):
    """3x3 halo conv whose only non-zero weight is the centre tap of channel 0: pixel (y, x) sees exactly x_m"""
    _, ops = _lib_ops()
    x = _xs(cuda)
    M = x.shape[0]
    H, W = 41, 80                                       # 3280 pixels >= 3203
    b = _bias(N, N + 2, cuda)
    w = torch.zeros(N, 8, 3, 3, device=cuda)
    w[:, 0, 1, 1] = 1.0
    pw = ops.pack_weight(w, b)
    src = torch.zeros(1, H, W, 8, dtype=torch.bfloat16, device=cuda)
    src.view(-1, 8)[:M, 0] = x
    out = torch.full((1, H, W, N), 7.0, dtype=torch.bfloat16, device=cuda)
    d = ops.gemm(pw, [src], out, image=(1, H, W), act=_acts(ops)[act])
    torch.cuda.synchronize()
    assert (d.bh, d.bw) == (16, 8)
    _check('halo N %d %s' % (N, act), act, out.view(-1, N)[:M], x.float()[:, None] + b[None, :])


@pytest.mark.parametrize('act2', ACTS)
def test_fused_tail_act2(cuda, act2):
    """fused trailing layer: main = x (no bias, no activation), w2 one-hot on column 0, b2 = 16 offsets: out3[m, i] =
    act2(x_m + b2[i]) in fp32 through the scalar gelu_erf"""
    _, ops = _lib_ops()
    x = _xs(cuda)
    M, N, n2 = x.shape[0], 32, 16
    w = torch.zeros(N, 8, device=cuda)
    w[:, 0] = 1.0
    pw = ops.pack_weight(w, None)
    xa = torch.zeros(M, 8, dtype=torch.bfloat16, device=cuda)
    xa[:, 0] = x
    w2 = torch.zeros(n2, N, device=cuda)
    w2[:, 0] = 1.0
    b2 = _bias(n2, 7, cuda)
    out = torch.zeros(M, N, dtype=torch.bfloat16, device=cuda)
    out3 = torch.zeros(M, n2, dtype=torch.float32, device=cuda)
    ops.gemm(pw, [xa], out, act=ops.ACT_NONE, tail=(w2, b2, _acts(ops)[act2]), tail_out=out3, skip_main=True)
    torch.cuda.synchronize()
    _check('fused tail act2 %s -> f32' % act2, act2, out3, x.float()[:, None] + b2[None, :])
