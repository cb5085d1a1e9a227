"""Pins the Swin window attention of oracle/pf_oracle.py (window_attention, shift_mask) against the reference's own
G2LBasicLayer / SwinTransformerBlock and writes tests/golden/window_case0.npz.
python -m oracle.make_golden_window  (needs $PATCHFUSION_REFERENCE)

Each case runs G2LBasicLayer.forward (its own pad-to-window arithmetic and shift-mask construction) with one
SwinTransformerBlock whose norm1 and attn.proj are nn.Identity(), whose MLP branch returns zeros and whose attn.qkv
returns the given qkv row of each token.  The block output minus its input is then the reference's window attention
(pad, cyclic roll, window partition, bias[relative_position_index], mask, softmax, reverse, roll back, crop) of that
qkv.  The input x carries the token's identity in channel 0 (index / 1024, 0 on the zero pad) so the qkv lookup
follows wherever the block moves the token.

Geometries: 14 x 19 (a 2 x 2 window grid with 10 pad rows and 5 pad columns) and 12 x 30 (one window row, 6 pad
columns), C 32 / 8 heads and C 64 / 16 heads, shift 0 and 6.  qkv holds bf16 values (what the kernel reads), stored as
fp16 (exact for them); pad tokens all hold one row, as Linear(0) = bias would give.
"""
import os
import sys

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import pf_oracle as po           # noqa: E402
from oracle import ref_harness as rh         # noqa: E402

OUT = os.path.join(ROOT, 'tests', 'golden', 'window_case0.npz')
WS = 12
# (H, W, C, heads, B)
GEOMS = ((14, 19, 32, 8, 2), (14, 19, 64, 16, 1), (12, 30, 32, 8, 1), (12, 30, 64, 16, 1))
SHIFTS = (0, WS // 2)


def tag(H, W, C):
    return '%dx%d_c%d' % (H, W, C)


def padded(H, W):
    return -(-H // WS) * WS, -(-W // WS) * WS


def case_inputs(H, W, C, heads, B, seed):
    """qkv [B, Hp * Wp, 3C] (bf16 values, |v| >= 2^-8 or 0 so that fp16 holds them exactly) and table [529, heads].
    qkv std 2 and a std-2 table: logits with std ~4, so the shift mask and the bias move the softmax visibly."""
    g = torch.Generator().manual_seed(seed)
    Hp, Wp = padded(H, W)
    q = (2 * torch.randn(B, Hp, Wp, 3 * C, generator=g)).to(torch.bfloat16).float()
    q = torch.where(q.abs() < 2.0 ** -8, torch.zeros_like(q), q)
    q[:, H:], q[:, :, W:] = q[0, 0, 0], q[0, 0, 0]          # every pad token holds one row (the qkv bias)
    table = (2 * torch.randn((2 * WS - 1) ** 2, heads, generator=g)).to(torch.bfloat16).float()
    return q.reshape(B, Hp * Wp, 3 * C), table


class _Lookup(nn.Module):
    """attn.qkv replaced: each token's qkv row, found from the identity in channel 0 of its (padded, rolled) input"""

    def __init__(self, rows):
        super().__init__()
        self.rows = rows

    def forward(self, x):
        return self.rows[torch.round(x[..., 0] * 1024).long()]


class _Zeros(nn.Module):
    def forward(self, x):
        return torch.zeros_like(x)


def reference_attention(qkv, table, H, W, C, heads, B, shift):
    """-> (the block's output minus its input [B, H * W, C] fp32, the layer's attn_mask [nW, 144, 144])"""
    from estimator.models.blocks.swin_layers import G2LBasicLayer
    Hp, Wp = padded(H, W)
    layer = G2LBasicLayer(dim=C, depth=2, num_heads=heads, window_size=WS).eval()
    blk = layer.blocks[0 if shift == 0 else 1]
    assert blk.shift_size == shift
    layer.blocks = nn.ModuleList([blk])
    grid = qkv.view(B, Hp, Wp, 3 * C)
    rows = torch.cat([grid[:1, H:H + 1, 0] if H < Hp else grid[:1, 0, W:W + 1], grid[:, :H, :W].reshape(1, -1, 3 * C)],
                     1)[0]                                   # row 0: the pad row; row 1 + t: token t (image-major)
    blk.norm1 = nn.Identity()
    blk.attn.qkv = _Lookup(rows)
    blk.attn.proj = nn.Identity()
    blk.mlp = _Zeros()
    blk.attn.relative_position_bias_table.data.copy_(table)
    seen = []
    fwd = blk.forward
    blk.forward = lambda x, m: (seen.append(m), fwd(x, m))[1]
    x = torch.zeros(B, H * W, C)
    x[..., 0] = (1 + torch.arange(B * H * W, dtype=torch.float32).view(B, H * W)) / 1024
    out, _, _ = layer(x, H, W)
    return (out.double() - x.double()).float(), seen[0]


def oracle_attention(qkv, table, H, W, C, heads, B, shift):
    """the oracle's composition of the same steps around pf_oracle.window_attention, fp32 -> [B, H * W, C]"""
    from patchfusion_b200.params import relative_position_index
    Hp, Wp = padded(H, W)
    x = qkv.view(B, Hp, Wp, 3 * C)
    if shift:
        x = torch.roll(x, shifts=(-shift, -shift), dims=(1, 2))
    mask = po.shift_mask(Hp, Wp, WS, 'cpu').repeat(B, 1, 1) if shift else None
    o = po.window_attention(po._windows(x, WS), table, relative_position_index(WS), heads, mask)
    o = po._unwindows(o, WS, Hp, Wp)
    if shift:
        o = torch.roll(o, shifts=(shift, shift), dims=(1, 2))
    return o[:, :H, :W].reshape(B, H * W, C)


def _rel(a, b):
    return ((a.double() - b.double()).abs().max() / b.double().abs().max()).item()


def main():
    rh._enter()
    torch.manual_seed(0)                      # the layer's own initialisation (overwritten) draws from the global RNG
    out = {}
    with torch.no_grad():
        for i, (H, W, C, heads, B) in enumerate(GEOMS):
            qkv, table = case_inputs(H, W, C, heads, B, seed=i)
            t = tag(H, W, C)
            out['qkv_' + t] = qkv.numpy().astype(np.float16)
            assert np.array_equal(out['qkv_' + t].astype(np.float32), qkv.numpy())
            out['table_' + t] = table.numpy()
            for shift in SHIFTS:
                ref, mask = reference_attention(qkv, table, H, W, C, heads, B, shift)
                mine = oracle_attention(qkv, table, H, W, C, heads, B, shift)
                e = _rel(mine, ref)
                print('%s shift %d: oracle vs reference rel-Linf %.2e' % (t, shift, e))
                assert e <= 1e-5, (t, shift, e)
                out['attn_%s_s%d' % (t, shift)] = ref.numpy()
                if shift:
                    assert torch.equal(mask, po.shift_mask(*padded(H, W), WS, 'cpu'))
                    out['mask_%dx%d' % (H, W)] = (mask != 0).numpy()
    np.savez_compressed(OUT, **out)
    print('wrote', OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
