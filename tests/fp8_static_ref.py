"""Static-scale FP8 (E4M3) references for fusion_precision = 'fp8_static': torch float8_e4m3fn emulations of
pf_quantize_e4m3_static and of the static conv's e4m3 output, bit for bit, and a static-FP8 Guided-Fusion U-Net for
oracle/pf_oracle.py.

The rule (include/pf_b200.h), in fp32:  r = 448 / amax (0 when amax == 0),  q = e4m3_rn(sat(v * r)),
scale = amax / 448, amax the conv input's calibrated value (one per conv, config `fusion_fp8_amax`).  torch's
float8_e4m3fn cast turns |x| > 464 into NaN, so the references clamp to +-448 first, as cvt.rn.satfinite does.
Weights keep fp8_ref's per-output-channel scales.  X.0 of a DoubleConv writes X.1's operand from its fp32 activation
(no bf16 rounding in between); every other U-Net activation is bf16 on the CUDA path.
"""
import contextlib

import torch
import torch.nn.functional as F

import fp8_ref

E4M3 = fp8_ref.E4M3


def ratio(amax):
    a = torch.tensor(float(amax), dtype=torch.float32)
    return torch.zeros(()) if a.item() == 0 else torch.tensor(448.0, dtype=torch.float32) / a


def scale(amax):
    a = torch.tensor(float(amax), dtype=torch.float32)
    return a / torch.tensor(448.0, dtype=torch.float32)


def quantize(v, amax):
    """v fp32 (any shape) -> float8_e4m3fn at the static ratio of amax, saturating"""
    r = ratio(amax).to(v.device)
    return (v.float() * r).clamp(-448.0, 448.0).to(E4M3)


def quantize_static_ref(srcs, src_c, amax):
    """pf_quantize_e4m3_static: bf16 NHWC maps [T,H,W,ld_i] -> uint8 [T,H,W,Kc] (sources back to back, 64-padded)"""
    out = []
    for s, c in zip(srcs, src_c):
        x = s[..., :c].float()
        seg = torch.zeros(x.shape[:3] + (fp8_ref.pad_to(c, 64),), dtype=torch.uint8, device=x.device)
        seg[..., :c] = quantize(x, amax).view(torch.uint8)
        out.append(seg)
    return torch.cat(out, -1)


def dequantize(q, amax):
    return q.float() * scale(amax).to(q.device)


def static_conv(x, w, bias, bn_scale, amax):
    """The static FP8 conv in fp32: x [T, C, H, W] as the kernel's input holds it (bf16 values, or X.0's fp32 output),
    quantized at amax; w per-channel e4m3 (BN scale folded when given); 3x3 pad 1"""
    if bn_scale is not None:
        w = w * bn_scale.view(-1, 1, 1, 1)
    qw, sw = fp8_ref.quantize(w, fp8_ref.group_amax(w))
    return F.conv2d(dequantize(quantize(x, amax), amax), fp8_ref.dequantize(qw, sw), bias, padding=1)


def layer_name(prefix):
    """oracle Weights prefix of a DoubleConv's container -> its name in params.FP8_LAYERS (without the .0 / .1)"""
    p = prefix[len('guided_fusion.'):] if prefix.startswith('guided_fusion.') else prefix
    parts = p.strip('.').split('.')
    if parts[0] == 'inc':
        return 'inc'
    if parts[0] == 'down_conv_list':
        return 'down%s' % parts[1]
    if parts[0] == 'up_conv_list':
        return 'up%d' % (int(parts[1]) + 1)
    if parts[0] == 'convs':
        return 'cv%s' % parts[1]
    raise KeyError(prefix)


def _double_conv_bn_static(table):
    def f(w, x):
        name = layer_name(w.prefix)
        x = x.to(torch.bfloat16).float()
        for j, (ci, bi) in enumerate(((0, 1), (3, 4))):
            p = 'double_conv.%d.' % bi
            s = w(p + 'weight') / torch.sqrt(w(p + 'running_var') + 1e-5)
            shift = w(p + 'bias') - w(p + 'running_mean') * s
            b = w('double_conv.%d.bias' % ci) * s + shift if w.has('double_conv.%d.bias' % ci) else shift
            x = F.relu(static_conv(x, w('double_conv.%d.weight' % ci), b, s, table['%s.%d' % (name, j)]))
        return x
    return f


def _double_conv_static(table):
    def f(w, x):
        name = layer_name(w.prefix)
        x = x.to(torch.bfloat16).float()
        x = F.relu(static_conv(x, w('double_conv.0.weight'), w('double_conv.0.bias'), None, table[name + '.0']))
        return F.relu(static_conv(x, w('double_conv.2.weight'), w('double_conv.2.bias'), None, table[name + '.1']))
    return f


@contextlib.contextmanager
def fp8_static_unet(table):
    """pf_oracle with the Guided-Fusion U-Net's 34 3x3 convs in emulated static FP8 at the calibration `table`;
    everything else as before"""
    from oracle import pf_oracle as po
    saved = po._double_conv_bn, po._double_conv
    po._double_conv_bn, po._double_conv = _double_conv_bn_static(table), _double_conv_static(table)
    try:
        yield po
    finally:
        po._double_conv_bn, po._double_conv = saved
