"""HBM-bound kernels vs torch fp32 / the oracle's restatements."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gpu_util import bf, check, from_nhwc, rb, to_nhwc

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(300)]


def _gen(seed):
    return torch.Generator(device='cuda').manual_seed(seed)


def test_layernorm(cuda):
    from patchfusion_b200 import ops
    g = _gen(0)
    for rows, C in [(1037, 384), (2074, 1024), (266, 64), (5, 32)]:
        x = torch.randn(rows, C, device=cuda, generator=g) * 3 + 1
        w, b = torch.randn(C, device=cuda, generator=g), torch.randn(C, device=cuda, generator=g)
        out = torch.zeros(rows, C, dtype=torch.bfloat16, device=cuda)
        ops.layernorm(x, w, b, 1e-6, out)
        check('layernorm %dx%d' % (rows, C), out, F.layer_norm(x, (C,), w, b, 1e-6), 1e-2)


@pytest.mark.parametrize('C', [1024, 100])
def test_layernorm_grouped(cuda, C):
    """pf_layernorm_grouped as the ViT's last blocks use it: B images of seq tokens, the cls row dropped (skip 1),
    npatch rows out per image.  x_ld and out_ld exceed C: NaN past C in x must not be read and the sentinel past C in
    the output must survive, as must the rows past B * npatch.  C = 1024 is the largest row, C = 100 ends in a partial
    group of 128 columns.  One token per image has mean 1e3 and std 1e-2: a one-pass E[x^2] - E[x]^2 variance
    cancels to noise there, the two-pass one keeps it."""
    import ctypes
    from patchfusion_b200 import ops
    g = _gen(7 + C)
    B, seq = 3, 1037
    npatch = seq - 1
    x_ld, out_ld, sentinel = C + 12, C + 20, -1024.0
    x = torch.full((B, seq, x_ld), float('nan'), device=cuda)
    x[..., :C] = torch.randn(B, seq, C, device=cuda, generator=g) * 3 + 1
    x[:, 5, :C] = 1e3 + 1e-2 * torch.randn(B, C, device=cuda, generator=g)
    w, b = 1 + 0.5 * torch.randn(C, device=cuda, generator=g), torch.randn(C, device=cuda, generator=g)
    out = torch.full((B * npatch + 8, out_ld), sentinel, dtype=torch.bfloat16, device=cuda)
    ops.call('pf_layernorm_grouped', x, x_ld, w, b, ctypes.c_float(1e-6), B, seq, 1, npatch, C, out, out_ld,
             ops.stream_ptr())
    torch.cuda.synchronize()
    ref = F.layer_norm(x[:, 1:, :C].double(), (C,), w.double(), b.double(), 1e-6).reshape(B * npatch, C)
    check('layernorm grouped C%d' % C, out[:B * npatch, :C], ref, 1e-2)
    o = out[:B * npatch, :C].view(B, npatch, C)
    check('layernorm grouped C%d mean 1e3 std 1e-2' % C, o[:, 4], ref.view(B, npatch, C)[:, 4], 2e-2)
    assert (out[:, C:] == sentinel).all() and (out[B * npatch:] == sentinel).all()


def test_patch_im2col_and_tokens(cuda):
    from patchfusion_b200 import ops
    g = _gen(1)
    B, H, W, D = 2, 392, 518, 384
    img = torch.rand(B, 3, H, W, device=cuda, generator=g)
    out = torch.zeros(B * 28 * 37, 592, dtype=torch.bfloat16, device=cuda)
    ops.call('pf_patch_im2col', img, B, H, W, out, 592, ops.stream_ptr())
    mean = torch.tensor([0.485, 0.456, 0.406], device=cuda).view(1, 3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225], device=cuda).view(1, 3, 1, 1)
    ref = F.unfold((img - mean) / std, 14, stride=14).transpose(1, 2).reshape(B * 28 * 37, 588)
    check('patch im2col', out[:, :588], ref, 5e-3)
    assert (out[:, 588:] == 0).all()
    patch = torch.randn(B, 1036, D, device=cuda, generator=g)
    cls, pos = torch.randn(D, device=cuda, generator=g), torch.randn(1037, D, device=cuda, generator=g)
    tok = torch.zeros(B, 1037, D, device=cuda)
    ops.call('pf_assemble_tokens', patch, cls, pos, B, 1036, D, tok, ops.stream_ptr())
    ref = torch.cat([cls.view(1, 1, D).expand(B, 1, D), patch], 1) + pos
    check('assemble tokens', tok, ref, 1e-6)


def test_resize_bilinear(cuda):
    from patchfusion_b200 import ops
    g = _gen(2)
    for (B, C, H, W, OH, OW) in [(2, 64, 14, 19, 28, 37), (1, 128, 224, 296, 392, 518), (2, 32, 49, 64, 56, 74),
                                 (1, 8, 196, 259, 224, 296), (1, 64, 56, 74, 56, 74), (2, 256, 112, 148, 224, 296),
                                 (1, 64, 98, 129, 112, 148), (3, 192, 60, 70, 61, 207)]:
        x = torch.randn(B, C, H, W, device=cuda, generator=g)
        out = torch.zeros(B, OH, OW, C + 16, dtype=torch.bfloat16, device=cuda)
        ops.resize_bilinear(to_nhwc(x), C, OH, OW, out, out_col0=8)
        ref = F.interpolate(rb(x), size=(OH, OW), mode='bilinear', align_corners=True)
        check('bilinear %dx%d->%dx%d' % (H, W, OH, OW), out[..., 8:8 + C].float().permute(0, 3, 1, 2), ref, 1e-2)
    x = torch.randn(2, 14, 19, 64, device=cuda, generator=g)
    out = torch.zeros(2, 28, 37, 64, device=cuda)
    ops.call('pf_resize_bilinear_f32', x, 2, 14, 19, 64, 28, 37, out, ops.stream_ptr())
    ref = F.interpolate(x.permute(0, 3, 1, 2), size=(28, 37), mode='bilinear', align_corners=True).permute(0, 2, 3, 1)
    check('bilinear f32', out, ref, 1e-5)


def test_roi_crop_zoom(cuda):
    from patchfusion_b200 import ops
    from torchvision.ops import roi_align
    g = _gen(3)
    P = (392, 518)
    boxes = torch.tensor([[0, 0, 129.5, 98.0], [64.75, 49.0, 194.25, 147.0], [388.5, 294.0, 518.0, 392.0],
                          [101.3, 250.7, 230.8, 348.7]], device=cuda)
    for (C, h, w) in [(64, 14, 19), (64, 224, 296), (32, 392, 518)]:
        f = torch.randn(1, C, h, w, device=cuda, generator=g)
        out = torch.zeros(4, h, w, C, dtype=torch.bfloat16, device=cuda)
        ops.roi_crop_zoom(to_nhwc(f), C, boxes, h / P[0], out)
        bxs = torch.cat([torch.zeros(4, 1, device=cuda), boxes], 1)
        ref = roi_align(rb(f), bxs, (h, w), h / P[0], aligned=True)
        check('roi crop-zoom %dx%d' % (h, w), from_nhwc(out, C), ref, 1e-2)
    d = torch.rand(392, 518, device=cuda, generator=g)
    out = torch.zeros(4, 392, 518, device=cuda)
    ops.roi_crop_zoom(d, 1, boxes, 1.0, out)
    bxs = torch.cat([torch.zeros(4, 1, device=cuda), boxes], 1)
    ref = roi_align(d[None, None], bxs, (392, 518), 1.0, aligned=True)[:, 0]
    check('roi crop-zoom fp32 depth', out, ref, 1e-5)


def test_maxpool_im2col_s2(cuda):
    from patchfusion_b200 import ops
    g = _gen(4)
    x = torch.randn(2, 32, 49, 64, device=cuda, generator=g)
    out = torch.zeros(2, 24, 32, 32, dtype=torch.bfloat16, device=cuda)
    ops.maxpool2(to_nhwc(x), 32, out)
    check('maxpool2', from_nhwc(out, 32), F.max_pool2d(rb(x), 2), 1e-6)
    x = torch.randn(2, 64, 28, 37, device=cuda, generator=g)
    out = torch.zeros(2 * 14 * 19, 9 * 64, dtype=torch.bfloat16, device=cuda)
    ops.call('pf_im2col_3x3_s2', to_nhwc(x), 2, 28, 37, 64, 64, out, ops.stream_ptr())
    ref = F.unfold(rb(x), 3, padding=1, stride=2)                       # [2, 64*9, 266] (c, tap)
    ref = ref.view(2, 64, 9, 266).permute(0, 3, 2, 1).reshape(2 * 266, 9 * 64)
    check('im2col 3x3 s2', out, ref, 1e-6)


def test_crop_resize_and_unet_input(cuda):
    from patchfusion_b200 import ops
    g = _gen(5)
    img = torch.rand(3, 1080, 1920, device=cuda, generator=g)
    origins = torch.tensor([[0, 0], [270, 480], [540, 960], [133, 777]], dtype=torch.int32, device=cuda)
    out = torch.zeros(4, 3, 392, 518, device=cuda)
    ops.call('pf_crop_resize', img, 1080, 1920, origins, 4, 540, 960, 392, 518, out, ops.stream_ptr())
    ref = torch.cat([F.interpolate(img[None, :, y:y + 540, x:x + 960], size=(392, 518), mode='bilinear',
                                   align_corners=True) for y, x in origins.tolist()])
    check('crop + resize', out, ref, 1e-5)
    cd, fd = torch.rand(4, 392, 518, device=cuda, generator=g), torch.rand(4, 392, 518, device=cuda, generator=g)
    u = torch.zeros(4, 392, 518, 8, dtype=torch.bfloat16, device=cuda)
    ops.call('pf_pack_unet_input', cd, fd, out, 4, 392, 518, u, 8, ops.stream_ptr())
    ref = torch.cat([cd[:, None], fd[:, None], out], 1)
    check('unet input', from_nhwc(u, 5), rb(ref), 1e-6)
    assert (u[..., 5:] == 0).all()


# ---------------------------------------------------------------------------------------------------- as the stages call
# The argument forms of csrc/pf_stage.cu: channel count pad8(C), row pitches wider than that.  The source columns
# [pad8(C), ld) and the images past the batch hold NaN (pf_maxpool2: 1e30, which fmaxf cannot drop), the outputs a
# sentinel; every value is compared with an fp64 reference on the bf16-rounded inputs.
SENTINEL = -77.0


def _poisoned_nhwc(x, C, ld, extra=1, fill=float('nan')):
    """fp32 [B, H, W, C] -> bf16 [B + extra, H, W, ld]: channels [C, pad8(C)) zero (as every producer writes them),
    [pad8(C), ld) and the `extra` images past the batch `fill`"""
    from patchfusion_b200 import ops
    B = x.shape[0]
    out = torch.full((B + extra,) + tuple(x.shape[1:3]) + (ld,), fill, dtype=torch.bfloat16, device=x.device)
    out[:B, ..., :ops.pad_to(C, 8)] = 0
    out[:B, ..., :C] = x.to(torch.bfloat16)
    return out


def _roi_align_fp64(feat, boxes, scale, images):
    """torchvision roi_align(aligned=True) with one sample per bin, output size = the map's, in fp64: feat [B, h, w, C],
    boxes [T, 4] (x1, y1, x2, y2), box t samples image images[t]"""
    _, h, w, C = feat.shape

    def taps(c, size):
        # roi_align's bilinear_interpolate: outside [-1, size] -> 0; clamp at 0; the last row / column has no neighbour
        valid = (c >= -1) & (c <= size)
        c = c.clamp_min(0)
        lo = c.floor().long().clamp_max(size - 1)
        edge = c.floor() >= size - 1
        hi = torch.where(edge, lo, lo + 1)
        fr = torch.where(edge, torch.zeros_like(c), c - lo)
        return lo, hi, fr, valid
    out = []
    for t in range(boxes.shape[0]):
        x1, y1, x2, y2 = (boxes[t].double() * scale - 0.5).tolist()
        ys = y1 + (torch.arange(h, dtype=torch.float64) + 0.5) * ((y2 - y1) / h)
        xs = x1 + (torch.arange(w, dtype=torch.float64) + 0.5) * ((x2 - x1) / w)
        yl, yh, fy, vy = taps(ys, h)
        xl, xh, fx, vx = taps(xs, w)
        f = feat[images[t]].double()
        fy, fx = fy.view(-1, 1, 1), fx.view(1, -1, 1)
        v = (1 - fy) * ((1 - fx) * f[yl][:, xl] + fx * f[yl][:, xh]) + fy * ((1 - fx) * f[yh][:, xl] + fx * f[yh][:, xh])
        out.append(v * (vy.view(-1, 1, 1) & vx.view(1, -1, 1)))
    return torch.stack(out)


# (x1, y1, x2, y2) at scale 0.5 on an 8 x 16 map: dyadic, so every sample coordinate is exact in fp32 and fp64
ROI_EDGE_BOXES = [
    [-2.0, -2.0, 30.0, 14.0],       # first samples exactly at -1
    [-1.5, 0.0, 30.5, 16.0],        # x samples in (-1, 0), y exactly at 0
    [2.0, 2.0, 34.0, 18.0],         # samples at size - 1 and exactly at size
    [1.0, 1.0, 41.0, 21.0],         # samples beyond size: zero
    [-4.0, -3.5, 28.0, 4.5],        # samples below -1: zero; then exactly -1
    [10.25, 3.5, 27.75, 12.25],     # fractional bins
    [0.75, 1.25, 31.5, 15.0],
]


@pytest.mark.parametrize('f32', [False, True], ids=['bf16', 'fp32'])
def test_roi_crop_zoom_batched_edges_poisoned(cuda, f32):
    import ctypes
    from patchfusion_b200 import ops
    g = _gen(11)
    B, h, w, C, ld, out_ld = 3, 8, 16, 20, 40, 48
    boxes = torch.tensor(ROI_EDGE_BOXES, device=cuda)
    T = boxes.shape[0]
    images = [2, 0, 1, 1, 2, 0, 1]
    tile_image = torch.tensor(images, dtype=torch.int32, device=cuda)
    if f32:                 # the coarse depth: [B, h, w] fp32, one channel; NaN in the image past the batch
        x = torch.rand(B, h, w, 1, device=cuda, generator=g) * 80
        feat = torch.cat([x[..., 0], torch.full((1, h, w), float('nan'), device=cuda)]).contiguous()
        out = torch.full((T + 1, h, w), SENTINEL, device=cuda)
        ops.call('pf_roi_crop_zoom_batched', feat, 1, h, w, 1, 1, tile_image, boxes, T, ctypes.c_float(0.5), out, 1, 0,
                 ops.stream_ptr())
        got, xin = out[:T, ..., None].double(), x.double()
    else:
        x = torch.randn(B, h, w, C, device=cuda, generator=g) * 4
        feat = _poisoned_nhwc(x, C, ld)
        out = torch.full((T + 1, h, w, out_ld), SENTINEL, dtype=torch.bfloat16, device=cuda)
        ops.call('pf_roi_crop_zoom_batched', feat, 0, h, w, ops.pad_to(C, 8), ld, tile_image, boxes, T,
                 ctypes.c_float(0.5), out, out_ld, 0, ops.stream_ptr())
        got, xin = out[:T, ..., :C].double(), rb(x).double()
        assert (out[:T, ..., C:ops.pad_to(C, 8)] == 0).all(), 'pad channels [C, pad8(C)) not zero'
        assert (out[:T, ..., ops.pad_to(C, 8):] == SENTINEL).all(), 'columns past pad8(C) written'
    assert (out[T:] == SENTINEL).all(), 'wrote past the last box'
    ref = _roi_align_fp64(xin.cpu(), boxes.cpu(), 0.5, images).to(cuda)
    assert (ref == 0).any() and (ref != 0).any()
    err = (got - ref).abs()
    if f32:
        tol = 1e-6 * xin.abs().max().item()
    else:
        # 1 bf16 ulp, plus the fp32 blend's own rounding where the value cancels to near zero
        tol = torch.pow(2.0, torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -126))) - 7) + 2.0 ** -22 * xin.abs().max()
    bad = (err > tol).nonzero()
    assert bad.numel() == 0, '%d values off by more than %s, first at %s: got %r want %r' % (
        bad.shape[0], 'the bound' if f32 else '1 bf16 ulp', bad[0].tolist(), got[tuple(bad[0])].item(),
        ref[tuple(bad[0])].item())
    print('roi crop-zoom %s: %d boxes at the roi_align edges, max |err| %.3e' % ('fp32' if f32 else 'bf16', T,
                                                                               err.max().item()))


def test_maxpool2_odd_poisoned(cuda):
    """odd H and W: the last row and column are not read (floor mode); they, the pad columns and the image past the
    batch hold 1e30, which wins any max it reaches"""
    from patchfusion_b200 import ops
    g = _gen(12)
    B, H, W, C, ld, out_ld = 2, 13, 17, 20, 40, 32
    x = torch.randn(B, H, W, C, device=cuda, generator=g)
    x[:, H - 1] = 1e30
    x[:, :, W - 1] = 1e30
    feat = _poisoned_nhwc(x, C, ld, fill=1e30)
    out = torch.full((B + 1, H // 2, W // 2, out_ld), SENTINEL, dtype=torch.bfloat16, device=cuda)
    ops.call('pf_maxpool2', feat, B, H, W, ops.pad_to(C, 8), ld, out, out_ld, ops.stream_ptr())
    ref = F.max_pool2d(rb(x).permute(0, 3, 1, 2), 2).permute(0, 2, 3, 1)
    assert torch.equal(out[:B, ..., :C].float(), ref)
    assert (out[:B, ..., C:ops.pad_to(C, 8)] == 0).all()
    assert (out[:B, ..., ops.pad_to(C, 8):] == SENTINEL).all() and (out[B:] == SENTINEL).all()


def test_im2col_3x3_s2_odd_poisoned(cuda):
    from patchfusion_b200 import ops
    g = _gen(13)
    B, H, W, C, ld = 2, 13, 17, 24, 40
    x = torch.randn(B, H, W, C, device=cuda, generator=g)
    feat = _poisoned_nhwc(x, C, ld)
    OH, OW = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    rows = B * OH * OW
    out = torch.full((rows + 4, 9 * C), SENTINEL, dtype=torch.bfloat16, device=cuda)
    ops.call('pf_im2col_3x3_s2', feat, B, H, W, C, ld, out, ops.stream_ptr())
    ref = F.unfold(rb(x).permute(0, 3, 1, 2), 3, padding=1, stride=2)          # [B, C * 9, OH * OW], (c, tap)
    ref = ref.view(B, C, 9, OH * OW).permute(0, 3, 2, 1).reshape(rows, 9 * C)
    assert torch.equal(out[:rows].float(), ref)
    assert (out[rows:] == SENTINEL).all()


def test_pack_unet_input_wide_poisoned(cuda):
    """ld 16: channels 0-4 are the bf16 roundings, 5-7 zero, [8, 16) and the tile past T keep the sentinel; the inputs'
    tile past T is NaN"""
    from patchfusion_b200 import ops
    g = _gen(14)
    T, H, W, ld = 3, 13, 17, 16
    nan = float('nan')
    cd, fd = torch.full((T + 1, H, W), nan, device=cuda), torch.full((T + 1, H, W), nan, device=cuda)
    rgb = torch.full((T + 1, 3, H, W), nan, device=cuda)
    cd[:T], fd[:T] = torch.rand(T, H, W, device=cuda, generator=g) * 80, torch.rand(T, H, W, device=cuda, generator=g) * 80
    rgb[:T] = torch.rand(T, 3, H, W, device=cuda, generator=g)
    u = torch.full((T + 1, H, W, ld), SENTINEL, dtype=torch.bfloat16, device=cuda)
    ops.call('pf_pack_unet_input', cd, fd, rgb, T, H, W, u, ld, ops.stream_ptr())
    ref = torch.cat([cd[:T, None], fd[:T, None], rgb[:T]], 1).permute(0, 2, 3, 1).to(torch.bfloat16)
    assert torch.equal(u[:T, ..., :5], ref)
    assert (u[:T, ..., 5:8] == 0).all()
    assert (u[:T, ..., 8:] == SENTINEL).all() and (u[T:] == SENTINEL).all()


def test_f32_to_bf16_rounding(cuda):
    """round to nearest even, as torch's conversion: ties both ways, +-0, subnormals (and their ties), the overflow
    to inf past the largest bf16, +-inf; NaN stays NaN"""
    from patchfusion_b200 import ops
    g = _gen(15)
    p = lambda e: 2.0 ** e                                                      # noqa: E731
    special = [1 + p(-8), 1 + 3 * p(-8), 1 + p(-8) + p(-20), -(1 + p(-8)), -(1 + 3 * p(-8)), 0.0, -0.0,
               p(-130), p(-133), p(-134), 3 * p(-134), -3 * p(-134), p(-149), p(-126) - p(-149), 1e-40,
               (2 - p(-8)) * p(127), (2 - p(-8) - p(-20)) * p(127), 3.4028234663852886e38, -3.4028234663852886e38,
               float('inf'), float('-inf'), 65504.0, 1.0 / 3]
    x = torch.cat([torch.tensor(special, device=cuda),
                   torch.randn(100003, device=cuda, generator=g) * torch.pow(10.0, torch.randint(
                       -30, 30, (100003,), device=cuda, generator=g).float()),
                   torch.tensor([float('nan'), -float('nan')], device=cuda)])
    n = x.numel()
    out = torch.full((n + 64,), SENTINEL, dtype=torch.bfloat16, device=cuda)
    ops.call('pf_f32_to_bf16', x, n, out, ops.stream_ptr())
    want = x.to(torch.bfloat16)
    got = out[:n]
    assert torch.isnan(got[-2:]).all(), 'NaN input must stay NaN'
    k = n - 2
    bad = (got[:k].view(torch.int16) != want[:k].view(torch.int16)).nonzero()
    assert bad.numel() == 0, '%d values differ, first %r -> %r (want %r)' % (
        bad.shape[0], x[bad[0]].item(), got[bad[0]].item(), want[bad[0]].item())
    assert (out[n:] == SENTINEL).all()


def test_swin_helpers(cuda):
    from patchfusion_b200 import ops
    g = _gen(6)
    H, W, C = 14, 19, 64
    Hp, Wp = 24, 24
    feat = torch.randn(1, C, H, W, device=cuda, generator=g)
    ape = torch.randn(H * W, C, device=cuda, generator=g)
    x = torch.zeros(H * W, C, device=cuda)
    ops.call('pf_g2l_embed', to_nhwc(feat), C, ape, H * W, C, x, ops.stream_ptr())
    xr = rb(feat).flatten(2).transpose(1, 2)[0] + ape
    check('g2l embed', x, xr, 1e-6)
    w, b = torch.randn(C, device=cuda, generator=g), torch.randn(C, device=cuda, generator=g)
    out = torch.full((Hp * Wp, C), 3.0, dtype=torch.bfloat16, device=cuda)
    ops.call('pf_swin_norm_pad', x, w, b, ops.C.c_float(1e-5), H, W, Hp, Wp, C, out, ops.stream_ptr())
    ref = F.pad(F.layer_norm(xr, (C,), w, b, 1e-5).view(H, W, C), (0, 0, 0, Wp - W, 0, Hp - H)).reshape(Hp * Wp, C)
    check('swin norm+pad', out, ref, 1e-2)
    y = torch.randn(Hp * Wp, C, device=cuda, generator=g)
    x2 = x.clone()
    ops.call('pf_swin_residual_crop', x2, y, H, W, Wp, C, ops.stream_ptr())
    check('swin residual crop', x2, x + y.view(Hp, Wp, C)[:H, :W].reshape(H * W, C), 1e-6)


def test_metric_tail(cuda):
    from patchfusion_b200 import ops
    from oracle import pf_oracle as po
    g = _gen(7)
    B, H, W, PH, PW, E = 2, 28, 37, 14, 19, 128
    a = torch.randn(B, E, H, W, device=cuda, generator=g)
    prev = torch.randn(B, E, PH, PW, device=cuda, generator=g)
    out = torch.zeros(B, H, W, E, dtype=torch.bfloat16, device=cuda)
    ops.call('pf_add_upsampled', to_nhwc(a), B, H, W, E, to_nhwc(prev), PH, PW, out, ops.stream_ptr())
    check('emb + up(prev)', from_nhwc(out, E), rb(a) + po.up(rb(prev), (H, W)), 1e-2)
    nA, nb = 16, 64
    A = F.softplus(torch.randn(B, H, W, 32, device=cuda, generator=g))
    bprev = F.softplus(torch.randn(B, PH, PW, nb, device=cuda, generator=g))
    bout = torch.zeros(B, H, W, nb, device=cuda)
    ops.call('pf_attractor', A, 32, nA, bprev, PH, PW, B, H, W, nb, 1, bout, ops.stream_ptr())
    bu = po.up(bprev.permute(0, 3, 1, 2), (H, W))
    An = A[..., :nA].permute(0, 3, 1, 2)
    ref = bu + po.inv_attractor(An.unsqueeze(2) - bu.unsqueeze(1)).mean(1)
    check('attractor', bout.permute(0, 3, 1, 2), ref, 1e-5)
    # log-binomial expectation
    Hh, Ww, BH, BW = 56, 74, 28, 37
    pt = F.softplus(torch.randn(B, Hh, Ww, 8, device=cuda, generator=g))
    bc = F.softplus(torch.randn(B, BH, BW, nb, device=cuda, generator=g)) * 3
    depth = torch.zeros(B, Hh, Ww, device=cuda)
    ops.call('pf_logbinom_depth', pt, 8, bc, BH, BW, B, Hh, Ww, nb, ops.C.c_float(0.0212), ops.C.c_float(50.0),
             depth, ops.stream_ptr())
    p4 = pt[..., :4].permute(0, 3, 1, 2)
    p, t = p4[:, :2] + 1e-4, p4[:, 2:] + 1e-4
    p = (p[:, 0] / (p[:, 0] + p[:, 1])).unsqueeze(1)
    t = (t[:, 0] / (t[:, 0] + t[:, 1])).unsqueeze(1)
    t = (50.0 - 0.0212) * t + 0.0212
    k = torch.arange(nb, dtype=torch.float32, device=cuda).view(1, nb, 1, 1)
    n_, k_ = torch.tensor(63.0, device=cuda) + 1e-7, k + 1e-7
    logc = n_ * torch.log(n_) - k_ * torch.log(k_) - (n_ - k_) * torch.log(n_ - k_ + 1e-7)
    y = logc + k * torch.log(p.clamp(1e-4, 1)) + (63 - k) * torch.log((1 - p).clamp(1e-4, 1))
    ref = (torch.softmax(y / t, 1) * po.up(bc.permute(0, 3, 1, 2), (Hh, Ww))).sum(1)
    check('log-binomial depth', depth, ref, 1e-4)


def test_stitch(cuda):
    from patchfusion_b200 import ops
    from oracle import pf_oracle as po
    g = _gen(8)
    CH, CW, th, tw = 784, 1036, 392, 518
    mask = torch.rand(th, tw, device=cuda, generator=g) + 1e-3
    tiles = torch.rand(5, th, tw, device=cuda, generator=g)
    org = [(0, 0), (0, 518), (392, 0), (392, 518), (196, 259)]
    num, den = torch.zeros(CH, CW, device=cuda), torch.zeros(CH, CW, device=cuda)
    o4 = torch.tensor(org[:4], dtype=torch.int32, device=cuda)
    o1 = torch.tensor(org[4:], dtype=torch.int32, device=cuda)
    ops.call('pf_stitch_accumulate', num, den, CH, CW, tiles, 4, th, tw, o4, mask, 0, 0, ops.stream_ptr())
    ops.call('pf_stitch_accumulate', num, den, CH, CW, tiles[4:], 1, th, tw, o1, mask, 0, 0, ops.stream_ptr())
    out = torch.zeros(CH, CW, device=cuda)
    ops.call('pf_stitch_finalize', num, den, CH * CW, out, ops.stream_ptr())
    # literal running average (oracle)
    cnt, acc = torch.zeros(CH, CW, device=cuda), torch.zeros(CH, CW, device=cuda)
    for (y, x), d in zip(org[:4], tiles[:4]):
        cnt[y:y + th, x:x + tw] = mask
        acc[y:y + th, x:x + tw] = d * mask
    ra = po.RunningAverage(acc, cnt)
    c2, a2 = torch.zeros(CH, CW, device=cuda), torch.zeros(CH, CW, device=cuda)
    c2[196:196 + th, 259:259 + tw] = mask
    a2[196:196 + th, 259:259 + tw] = tiles[4] * mask
    ra.update(a2, c2)
    check('stitch (regular)', out, ra.avg, 1e-5)
    # resize + a random (nearest-upsampled) tile
    OH, OW, uh, uw = 1080, 1920, 540, 960
    n2, d2 = torch.zeros(OH, OW, device=cuda), torch.zeros(OH, OW, device=cuda)
    ops.call('pf_stitch_resize', num, den, CH, CW, OH, OW, n2, d2, ops.stream_ptr())
    mask2 = torch.rand(uh, uw, device=cuda, generator=g) + 1e-3
    o = torch.tensor([[100, 333]], dtype=torch.int32, device=cuda)
    ops.call('pf_stitch_accumulate', n2, d2, OH, OW, tiles[:1], 1, th, tw, o, mask2, uh, uw, ops.stream_ptr())
    out2 = torch.zeros(OH, OW, device=cuda)
    ops.call('pf_stitch_finalize', n2, d2, OH * OW, out2, ops.stream_ptr())
    ra.resize((OH, OW))
    upd = F.interpolate(tiles[:1, None], (uh, uw))[0, 0]
    c3, a3 = torch.zeros(OH, OW, device=cuda), torch.zeros(OH, OW, device=cuda)
    c3[100:100 + uh, 333:333 + uw] = mask2
    a3[100:100 + uh, 333:333 + uw] = upd * mask2
    ra.update(a3, c3)
    check('stitch (resize + random tile)', out2, ra.avg, 1e-5)


def test_stitch_gather_deterministic(cuda):
    """pf_stitch_gather (the product path's stitch): equals the literal sequential RunningAverage to fp32 rounding, is
    bit-identical under any permutation of where the predictions sit (slot table = the gathered per-rank blocks), and
    continues from resized base canvases for the random phase."""
    from patchfusion_b200 import ops
    from patchfusion_b200.parallel import slot_table
    from oracle import pf_oracle as po
    g = _gen(18)
    CH, CW, th, tw = 784, 1036, 392, 518
    mask = torch.rand(th, tw, device=cuda, generator=g) + 1e-3
    org = [(0, 0), (0, 518), (392, 0), (392, 518), (0, 259), (392, 259), (196, 0), (196, 518), (196, 259)]
    n = len(org)
    tiles = torch.rand(n, th, tw, device=cuda, generator=g)

    def gather(preds, slots, up=(0, 0), msk=mask, base=(None, None), shape=(CH, CW), want=('num', 'den', 'avg')):
        tab = torch.tensor([(y, x, s_) for (y, x), s_ in zip(org_l, slots)], dtype=torch.int32, device=cuda)
        o = {k: torch.empty(shape, device=cuda) for k in want}
        ops.call('pf_stitch_gather', preds, tab, len(slots), th, tw, msk, up[0], up[1], base[0], base[1], shape[0],
                 shape[1], o.get('num'), o.get('den'), o.get('avg'), ops.stream_ptr())
        return o

    org_l = org
    a = gather(tiles, list(range(n)))
    # sharded layout: world 4, blocks of ceil(9/4)=3 rows, padding rows NaN
    world, per = 4, 3
    full = torch.full((world * per, th, tw), float('nan'), device=cuda)
    slots = slot_table(n, world)
    for i, s_ in enumerate(slots):
        full[s_] = tiles[i]
    b = gather(full, slots)
    assert torch.equal(a['avg'], b['avg']) and torch.equal(a['num'], b['num']) and torch.equal(a['den'], b['den'])
    cnt, acc = torch.zeros(CH, CW, device=cuda), torch.zeros(CH, CW, device=cuda)
    for (y, x), d in zip(org[:4], tiles[:4]):
        cnt[y:y + th, x:x + tw] = mask
        acc[y:y + th, x:x + tw] = d * mask
    ra = po.RunningAverage(acc, cnt)
    for (y, x), d in zip(org[4:], tiles[4:]):
        c2, a2 = torch.zeros(CH, CW, device=cuda), torch.zeros(CH, CW, device=cuda)
        c2[y:y + th, x:x + tw] = mask
        a2[y:y + th, x:x + tw] = d * mask
        ra.update(a2, c2)
    check('stitch gather (regular, 9 tiles)', a['avg'], ra.avg, 1e-5)
    # random phase on top of the resized canvases
    OH, OW, uh, uw = 1080, 1920, 540, 960
    n2, d2 = torch.empty(OH, OW, device=cuda), torch.empty(OH, OW, device=cuda)
    ops.call('pf_stitch_resize', a['num'], a['den'], CH, CW, OH, OW, n2, d2, ops.stream_ptr())
    mask2 = torch.rand(uh, uw, device=cuda, generator=g) + 1e-3
    org_l = [(100, 333), (400, 333), (17, 333)]
    r = gather(tiles[:3].contiguous(), [0, 1, 2], up=(uh, uw), msk=mask2, base=(n2, d2), shape=(OH, OW), want=('avg',))
    ra.resize((OH, OW))
    for (y, x), d in zip(org_l, F.interpolate(tiles[:3, None], (uh, uw))[:, 0]):
        c3, a3 = torch.zeros(OH, OW, device=cuda), torch.zeros(OH, OW, device=cuda)
        c3[y:y + uh, x:x + uw] = mask2
        a3[y:y + uh, x:x + uw] = d * mask2
        ra.update(a3, c3)
    check('stitch gather (resize + 3 random tiles)', r['avg'], ra.avg, 1e-5)


def test_ingest_and_u16_writer(cuda):
    """the callers either side of the path (SURVEY §8f): bicubic align_corners ingest and the uint16 depth writer"""
    from patchfusion_b200 import imageio
    g = torch.Generator().manual_seed(9)
    img = torch.randint(0, 256, (270, 480, 3), generator=g, dtype=torch.uint8)
    got = imageio.ingest(img.numpy(), (1080, 1920), cuda, bgr=True)
    rgb = img.numpy()[:, :, ::-1].copy()
    ref = F.interpolate(torch.tensor(rgb / 255.0).unsqueeze(0).permute(0, 3, 1, 2), (1080, 1920), mode='bicubic',
                        align_corners=True).float()
    assert got.shape == (1, 3, 1080, 1920)
    assert (got.cpu() - ref).abs().max().item() < 1e-4
    d = torch.rand(784, 1036, generator=g) * 80
    u = imageio.depth_to_u16(d.to(cuda)[None, None], (1080, 1920))
    want = (F.interpolate(d[None, None], (1080, 1920))[0, 0].numpy() * 256).astype('uint16')
    assert u.dtype == torch.uint16 and (u.cpu().numpy().astype(np.int64) - want.astype(np.int64)).__abs__().max() <= 1
