"""Static-scale FP8 (E4M3) emulation of the DPT decoders for dpt_precision = 'fp8_static', on oracle/pf_oracle.py.

The 19 convs of params.DPT_FP8_CONVS of each branch read their input as the CUDA path does: the bf16 value quantized
at the conv's calibrated amax (fp8_static_ref.quantize), against per-output-channel e4m3 weights (fp8_ref); the RCU
conv2 operand is conv1's fp32 ReLU output quantized directly (the kernel writes it from the accumulator).  Everything
else is the oracle's fp32 arithmetic.
"""
import contextlib

import torch
import torch.nn.functional as F

import fp8_ref
import fp8_static_ref as sref


def weight_e4m3(w):
    qw, sw = fp8_ref.quantize(w.float(), fp8_ref.group_amax(w))
    return fp8_ref.dequantize(qw, sw)


def conv_e4m3_f64(q, amax, w, bias):
    """fp64 3x3 conv (pad 1) of the dequantized e4m3 NHWC map q (uint8 [T, H, W, >= C]) and the dequantized weight;
    NHWC out"""
    C = w.shape[1]
    a = q[..., :C].view(sref.E4M3).double() * sref.scale(amax).double().to(q.device)
    y = F.conv2d(a.permute(0, 3, 1, 2), weight_e4m3(w).double(), None if bias is None else bias.double(), padding=1)
    return y.permute(0, 2, 3, 1)


def _branch(prefix):
    return prefix.split('_branch.')[0].split('.')[-1]


def _make_weights(po, table):
    class W8(po.Weights):
        """the oracle's Weights, with the covered convs of a depth head's scratch in static FP8"""
        def sub(self, p):
            return W8(self.sd, self.prefix + p)

        def conv(self, name, x, stride=1, padding=0):
            key = (self.prefix + name).split('depth_head.scratch.')[-1]
            full = '%s.%s' % (_branch(self.prefix), key)
            if 'depth_head.scratch.' not in self.prefix + name or full not in table:
                return super().conv(name, x, stride=stride, padding=padding)
            b = self(name + '.bias') if self.has(name + '.bias') else None
            v = x if key.endswith('conv2') else x.to(torch.bfloat16).float()   # conv2 reads conv1's fp32 output
            a = sref.dequantize(sref.quantize(v, table[full]), table[full])
            return F.conv2d(a, weight_e4m3(self(name + '.weight')), b, stride=stride, padding=padding)
    return W8


@contextlib.contextmanager
def fp8_static_dpt(table):
    """pf_oracle with the 19 covered DPT convs of both branches in emulated static FP8 at the calibration `table`;
    everything else as before"""
    from oracle import pf_oracle as po
    saved = po.dpt_head
    W8 = _make_weights(po, table)

    def dpt_head(w, feats, gh, gw):
        return saved(W8(w.sd, w.prefix), feats, gh, gw)
    po.dpt_head = dpt_head
    try:
        yield po
    finally:
        po.dpt_head = saved
