"""Static-scale FP8 (E4M3) references for vit_precision = 'fp8_static': a torch restatement of pf_layernorm_e4m3, the
E4M3 linear in fp64 over dequantized operands, and a DINOv2 block for oracle/pf_oracle.py with qkv, fc1 and fc2 on
emulated static FP8.

The rule is fusion_precision 'fp8_static''s (tests/fp8_static_ref.py): r = 448 / amax, q = e4m3_rn(sat(v * r)),
scale = amax / 448, amax the linear input's calibrated value (config `vit_fp8_amax`).  Weights keep fp8_ref's
per-output-channel scales.  LN1 / LN2 quantize their fp32 affine value and fc1 its fp32 GELU output, with no bf16
rounding in between; proj stays bf16.
"""
import contextlib

import torch
import torch.nn.functional as F

import fp8_ref
import fp8_static_ref as sref

E4M3 = fp8_ref.E4M3


def layernorm_f32(x, w, b, eps):
    """pf_layernorm's fp32 statistics (mean, centred variance) and its affine step fma((x - mean) * rstd, w, b),
    restated in torch: the fused multiply-add is taken in fp64 and rounded once.  The kernel sums in another order and
    uses rsqrt, so a few values may differ in the last fp32 bit."""
    x = x.float()
    C = x.shape[-1]
    mean = x.sum(-1, keepdim=True) / C
    c = x - mean
    rstd = torch.rsqrt((c * c).sum(-1, keepdim=True) / C + eps)
    t = c * rstd
    return (t.double() * w.double() + b.double()).float()


def layernorm_e4m3(x, w, b, eps, amax):
    """pf_layernorm_e4m3: uint8 [rows, C]"""
    return sref.quantize(layernorm_f32(x, w, b, eps), amax).view(torch.uint8)


def weight_e4m3(w):
    """per-output-channel e4m3 weights, dequantized (pf_pack_weight_e4m3 over a Linear weight [N, K])"""
    qw, sw = fp8_ref.quantize(w.float(), fp8_ref.group_amax(w))
    return fp8_ref.dequantize(qw, sw)


def linear_e4m3_f64(q, amax, w, bias):
    """fp64 linear of the dequantized e4m3 input q (uint8 [M, K], static scale of amax) and the dequantized weight"""
    a = q.view(E4M3).double() * sref.scale(amax).double().to(q.device)
    return F.linear(a, weight_e4m3(w).double(), None if bias is None else bias.double())


def _name(prefix):
    """oracle Weights prefix of a ViT block -> ('coarse' | 'fine', block index)"""
    branch = prefix.split('_branch.')[0].split('.')[-1]
    return branch, int(prefix.rstrip('.').split('.')[-1])


def _vit_block_static(table):
    def f(w, x, heads):
        branch, i = _name(w.prefix)
        am = {k: table['%s.%d.%s' % (branch, i, k)] for k in ('qkv', 'fc1', 'fc2')}

        def lin(name, v, amax):
            a = sref.dequantize(sref.quantize(v, amax), amax)
            return F.linear(a, weight_e4m3(w(name + '.weight')), w(name + '.bias'))
        B, N, D = x.shape
        hd = D // heads
        h = w.ln('norm1', x, 1e-6)
        qkv = lin('attn.qkv', h, am['qkv']).reshape(B, N, 3, heads, hd).permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0] * hd ** -0.5, qkv[1], qkv[2]
        a = (q @ k.transpose(-2, -1)).softmax(dim=-1)
        h = (a @ v).transpose(1, 2).reshape(B, N, D)
        x = x + w('ls1.gamma') * w.linear('attn.proj', h)
        h = w.ln('norm2', x, 1e-6)
        h = lin('mlp.fc2', F.gelu(lin('mlp.fc1', h, am['fc1'])), am['fc2'])
        return x + w('ls2.gamma') * h
    return f


@contextlib.contextmanager
def fp8_static_vit(table):
    """pf_oracle with the qkv, fc1 and fc2 linears of both DINOv2 encoders in emulated static FP8 at the calibration
    `table`; everything else as before"""
    from oracle import pf_oracle as po
    saved = po.vit_block
    po.vit_block = _vit_block_static(table)
    try:
        yield po
    finally:
        po.vit_block = saved
