"""FP8 (E4M3) references for fusion_precision = 'fp8': torch float8_e4m3fn emulations of pf_pack_weight_e4m3 and
pf_quantize_e4m3_tiles, bit for bit, and an FP8-emulating Guided-Fusion U-Net for oracle/pf_oracle.py.

The rounding rule (include/pf_b200.h), in fp32:  amax = max |v| over the group,  r = 448 / amax (0 when amax == 0),
q = e4m3_rn(v * r),  scale = amax / 448.  Weights: one group per output channel, BatchNorm folded first.  Activations:
one group per tile (U-Net batch index) over all of a conv's input channels.  The emulated conv computes, in fp32,
conv(dequant(q_x), dequant(q_w)) with dequant(q) = float(q) * scale.
"""
import contextlib

import torch
import torch.nn.functional as F

E4M3 = torch.float8_e4m3fn
E4M3_MAX = 448.0


def pad_to(n, m):
    return (n + m - 1) // m * m


def _ratio(amax):
    amax = amax.float()
    return torch.where(amax == 0, torch.zeros_like(amax), torch.full_like(amax, E4M3_MAX) / amax)


def _scale(amax):
    # a tensor divisor: torch divides by a Python scalar as a multiplication by its reciprocal, which rounds differently
    amax = amax.float()
    return amax / torch.full_like(amax, E4M3_MAX)


def quantize(v, amax):
    """v fp32 [G, ...], amax fp32 [G] -> (q float8_e4m3fn like v, scale fp32 [G])"""
    r = _ratio(amax).view(-1, *([1] * (v.dim() - 1)))
    return (v.float() * r).to(E4M3), _scale(amax)


def dequantize(q, scale):
    return q.float() * scale.view(-1, *([1] * (q.dim() - 1)))


def group_amax(v):
    """max |v| per leading index, NaN-propagating like the kernels"""
    a = v.float().abs().flatten(1)
    m = a.amax(1)
    return torch.where(torch.isnan(a).any(1), torch.full_like(m, float('nan')), m)


def pack_weight_e4m3_ref(w, src_c=None, scale=None, n_pad=None):
    """pf_pack_weight_e4m3: w fp32 [N, C, 3, 3] (or [N, C]) -> (panel uint8 [n_pad, Ktot], s_w fp32 [N])"""
    w = w.float()
    N = w.shape[0]
    taps = 1 if w.dim() == 2 else w.shape[2] * w.shape[3]
    w = w.reshape(N, w.shape[1], taps)
    if scale is not None:
        w = w * scale.float().view(N, 1, 1)
    src_c = [w.shape[1]] if src_c is None else list(src_c)
    q, s_w = quantize(w, group_amax(w))
    qb = q.view(torch.uint8)
    segs, c0 = [], 0
    for c in src_c:
        cp = pad_to(c, 64)
        seg = torch.zeros((N, taps, cp), dtype=torch.uint8, device=w.device)
        seg[:, :, :c] = qb[:, c0:c0 + c, :].permute(0, 2, 1)
        segs.append(seg.reshape(N, taps * cp))
        c0 += c
    panel = torch.cat(segs, 1)
    if n_pad is not None and n_pad > N:
        panel = torch.cat([panel, torch.zeros((n_pad - N, panel.shape[1]), dtype=torch.uint8, device=w.device)])
    return panel, s_w


def quantize_tiles_ref(srcs, src_c):
    """pf_quantize_e4m3_tiles: bf16 NHWC maps [T,H,W,ld_i] -> (uint8 [T,H,W,Kc], s_a fp32 [T])"""
    xs = [s[..., :c].float() for s, c in zip(srcs, src_c)]
    T = xs[0].shape[0]
    amax = group_amax(torch.cat([x.reshape(T, -1) for x in xs], 1))
    out = []
    for x, c in zip(xs, src_c):
        q, _ = quantize(x, amax)
        seg = torch.zeros(x.shape[:3] + (pad_to(c, 64),), dtype=torch.uint8, device=x.device)
        seg[..., :c] = q.view(torch.uint8)
        out.append(seg)
    return torch.cat(out, -1), _scale(amax)


def fp8_conv(x, w, bias, scale=None):
    """The FP8 conv in fp32: x [T, C, H, W], w [N, C, 3, 3] (BN scale folded when given), per-tile and per-channel
    scales, 3x3 pad 1.  x is rounded to bf16 first: the CUDA path stores every U-Net activation in bf16, and
    quantizing the fp32 value instead would move some elements across an e4m3 rounding boundary (one e4m3 step is
    6 % of the value)."""
    if scale is not None:
        w = w * scale.view(-1, 1, 1, 1)
    x = x.to(torch.bfloat16).float()
    qw, sw = quantize(w, group_amax(w))
    qx, sx = quantize(x, group_amax(x))
    return F.conv2d(dequantize(qx, sx), dequantize(qw, sw), bias, padding=1)


def _double_conv_bn_fp8(w, x):
    for ci, bi in ((0, 1), (3, 4)):
        p = 'double_conv.%d.' % bi
        s = w(p + 'weight') / torch.sqrt(w(p + 'running_var') + 1e-5)
        shift = w(p + 'bias') - w(p + 'running_mean') * s
        b = w('double_conv.%d.bias' % ci) * s + shift if w.has('double_conv.%d.bias' % ci) else shift
        x = F.relu(fp8_conv(x, w('double_conv.%d.weight' % ci), b, s))
    return x


def _double_conv_fp8(w, x):
    x = F.relu(fp8_conv(x, w('double_conv.0.weight'), w('double_conv.0.bias')))
    return F.relu(fp8_conv(x, w('double_conv.2.weight'), w('double_conv.2.bias')))


@contextlib.contextmanager
def fp8_unet():
    """pf_oracle with the Guided-Fusion U-Net's 3x3 convs (inc, down_conv_list, up_conv_list, convs) in emulated FP8;
    everything else (fusion_conv_list, G2L, the head, the branches) as before"""
    from oracle import pf_oracle as po
    saved = po._double_conv_bn, po._double_conv
    po._double_conv_bn, po._double_conv = _double_conv_bn_fp8, _double_conv_fp8
    try:
        yield po
    finally:
        po._double_conv_bn, po._double_conv = saved
