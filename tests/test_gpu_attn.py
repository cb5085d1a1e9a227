"""pf_attention (wgmma flash-style) and pf_window_attention vs torch fp32."""
import pytest
import torch
import torch.nn.functional as F

from attn_ref import FP64_TOL
from gpu_util import bf, check, rb

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]


@pytest.mark.parametrize('B,seq,heads', [(1, 1037, 6), (2, 1037, 16), (1, 200, 2), (3, 128, 1)])
def test_attention(cuda, B, seq, heads):
    from patchfusion_b200 import ops
    g = torch.Generator(device='cuda').manual_seed(seq + heads)
    D = heads * 64
    seq_pad = ops.pad_to(seq, 8)
    q = torch.randn(B, seq, heads, 64, device=cuda, generator=g)
    k = torch.randn(B, seq, heads, 64, device=cuda, generator=g)
    v = torch.randn(B, seq, heads, 64, device=cuda, generator=g)
    qk = torch.cat([q.reshape(B * seq, D), k.reshape(B * seq, D)], 1).to(torch.bfloat16).contiguous()
    vt = torch.zeros(B * D, seq_pad, dtype=torch.bfloat16, device=cuda)
    vt.view(B, D, seq_pad)[:, :, :seq] = bf(v.reshape(B, seq, D).permute(0, 2, 1))
    out = torch.zeros(B * seq, D, dtype=torch.bfloat16, device=cuda)
    ops.attention(qk, vt, B, seq, seq_pad, heads, 0.125, out)
    torch.cuda.synchronize()
    qq, kk, vv = [rb(t).permute(0, 2, 1, 3) for t in (q, k, v)]
    a = (qq @ kk.transpose(-1, -2) * 0.125).softmax(-1)
    ref = (a @ vv).permute(0, 2, 1, 3).reshape(B * seq, D)
    check('attention B%d seq%d h%d' % (B, seq, heads), out, ref, FP64_TOL)


@pytest.mark.parametrize('H,W,C,heads,shift', [(14, 19, 64, 32, 0), (14, 19, 64, 32, 6), (28, 37, 256, 32, 6),
                                               (56, 74, 128, 8, 6), (24, 36, 32, 8, 0), (30, 50, 256, 8, 6)])
def test_window_attention(cuda, H, W, C, heads, shift):
    _window_attention(cuda, H, W, C, heads, shift, 1.0, 1.0)


@pytest.mark.parametrize('H,W,C,heads', [(14, 19, 64, 4), (28, 37, 256, 8)])
@pytest.mark.parametrize('shift', [0, 6])
def test_window_attention_peaky(cuda, H, W, C, heads, shift):
    """qkv x8 and a bias table with std 5: logits with std in the tens, so the running maximum moves late and far and
    the kernel's rescale-when-the-maximum-moves branch does real work"""
    _window_attention(cuda, H, W, C, heads, shift, 8.0, 5.0)


def _window_attention(cuda, H, W, C, heads, shift, qkv_scale, table_std):
    from patchfusion_b200 import ops
    import math
    from oracle import pf_oracle as po
    ws = 12
    Hp, Wp = math.ceil(H / ws) * ws, math.ceil(W / ws) * ws
    g = torch.Generator(device='cuda').manual_seed(H * W + C)
    qkv = torch.randn(Hp * Wp, 3 * C, device=cuda, generator=g) * qkv_scale
    table = torch.randn(529, heads, device=cuda, generator=g) * table_std
    out = torch.zeros(Hp * Wp, C, dtype=torch.bfloat16, device=cuda)
    ops.call('pf_window_attention', bf(qkv).contiguous(), table, Hp, Wp, C, heads, shift, out, ops.stream_ptr())
    torch.cuda.synchronize()
    # torch reference in the reference's own formulation (roll -> windows -> attention -> reverse -> roll back)
    from patchfusion_b200.params import relative_position_index
    hd = C // heads
    x = rb(qkv).view(1, Hp, Wp, 3 * C)
    if shift:
        x = torch.roll(x, shifts=(-shift, -shift), dims=(1, 2))
    win = po._windows(x, ws)
    nW, N = win.shape[0], ws * ws
    t = win.reshape(nW, N, 3, heads, hd).permute(2, 0, 3, 1, 4)
    q, k, v = t[0] * hd ** -0.5, t[1], t[2]
    a = q @ k.transpose(-1, -2)
    idx = relative_position_index().to(cuda).view(-1)
    a = a + table[idx].view(N, N, heads).permute(2, 0, 1).unsqueeze(0)
    if shift:
        a = a + po.shift_mask(Hp, Wp, ws, cuda).unsqueeze(1)
    o = (a.softmax(-1) @ v).transpose(1, 2).reshape(nW, N, C)
    o = po._unwindows(o, ws, Hp, Wp)
    if shift:
        o = torch.roll(o, shifts=(shift, shift), dims=(1, 2))
    check('window attention %dx%d C%d h%d s%d x%g' % (H, W, C, heads, shift, qkv_scale), out, o.reshape(Hp * Wp, C), 1e-2)
