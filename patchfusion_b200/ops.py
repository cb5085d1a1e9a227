"""Thin Python wrappers over the C ABI: weight packing and one function per kernel family.

Tensors are torch CUDA tensors used as typed device buffers: activations bf16 NHWC (`[B, H, W, ld]`, logical
channel count tracked by the caller), token matrices `[rows, ld]`, fp32 where include/pf_b200.h says so.
"""
import ctypes as C

import numpy as np
import torch

from . import lib
from .lib import ACT_GELU, ACT_NONE, ACT_RELU, ACT_SOFTPLUS, GemmDesc, call, stream_ptr  # noqa: F401


def pad_to(n, m):
    return (n + m - 1) // m * m


class PackedWeight:
    """bf16 K-major weight panel for pf_gemm + fp32 bias.  An FP8 layer (pack_weight_e4m3) also has an e4m3 panel `w8`
    [N_pad, Ktot] (uint8 storage) and its per-output-channel scales `w_scale` [N]; its bf16 `w` may be None."""
    w8 = None
    w_scale = None

    def __init__(self, w, bias, N, src_c, taps, ps=1, ps_cout=0):
        self.w, self.bias, self.N, self.src_c, self.taps = w, bias, N, list(src_c), taps
        self.Ktot = w.shape[1]
        self.ps, self.ps_cout = ps, ps_cout


def n_pad_for(N):
    """rows of the packed panel: what pf_gemm's automatic block_n choice will read (multiple of block_n)."""
    n32 = pad_to(N, 32)
    if n32 <= 256:
        return n32
    best, bn = None, None
    for c in range(256, 127, -32):
        pad = pad_to(N, c) - N
        if best is None or pad < best:
            best, bn = pad, c
    return pad_to(N, bn)


def pack_weight(weight, bias=None, src_c=None, scale=None, shift=None):
    """weight: fp32 [N, C, kh, kw] or [N, C] on the GPU.  `scale/shift` fold an eval-mode BatchNorm:
    y = scale * conv(x) + shift."""
    weight = weight.float().contiguous()
    N = weight.shape[0]
    taps = 1 if weight.dim() == 2 else weight.shape[2] * weight.shape[3]
    assert taps in (1, 9)
    ctot = weight.shape[1]
    src_c = [ctot] if src_c is None else list(src_c)
    assert sum(src_c) == ctot and 1 <= len(src_c) <= 3
    Ktot = sum(taps * pad_to(c, 64) for c in src_c)
    n_pad = n_pad_for(N)
    dst = torch.empty((n_pad, Ktot), dtype=torch.bfloat16, device=weight.device)
    sc = (C.c_int32 * 3)(*(src_c + [0] * (3 - len(src_c))))
    scale_t = scale.float().contiguous() if scale is not None else None
    call('pf_pack_weight', weight, N, n_pad, len(src_c), sc, taps, scale_t, dst, stream_ptr())
    b = None
    if bias is not None or shift is not None:
        b = torch.zeros(N, dtype=torch.float32, device=weight.device)
        if bias is not None:
            b += bias.float() * (scale.float() if scale is not None else 1.0)
        if shift is not None:
            b += shift.float()
    return PackedWeight(dst, b, N, src_c, taps)


def pack_weight_e4m3(weight, bias=None, src_c=None, scale=None, shift=None, keep_bf16=False):
    """pack_weight's panel as e4m3 with one fp32 scale per output channel (pf_pack_weight_e4m3; the rounding rule is
    in include/pf_b200.h).  keep_bf16: also keep the bf16 panel (a conv that may run through the fused resample)."""
    pw = pack_weight(weight, bias, src_c=src_c, scale=scale, shift=shift)
    weight = weight.float().contiguous()
    w8 = torch.empty(pw.w.shape, dtype=torch.uint8, device=weight.device)
    s_w = torch.empty(pw.N, dtype=torch.float32, device=weight.device)
    sc = (C.c_int32 * 3)(*(pw.src_c + [0] * (3 - len(pw.src_c))))
    scale_t = scale.float().contiguous() if scale is not None else None
    call('pf_pack_weight_e4m3', weight, pw.N, pw.w.shape[0], len(pw.src_c), sc, pw.taps, scale_t, w8, s_w, stream_ptr())
    pw.w8, pw.w_scale = w8, s_w
    if not keep_bf16:
        pw.w = None
    return pw


def quantize_e4m3_tiles(srcs, src_c=None, out=None, s_a=None):
    """srcs: bf16 NHWC maps [T,H,W,ld_i] (logical channels src_c[i], default the last dim).  Returns (q, s_a): the
    e4m3 map [T,H,W,Kc] (uint8 storage, sources back to back, each padded to 64 channels) and the fp32 tile scales [T]
    (pf_quantize_e4m3_tiles)."""
    T, H, W = srcs[0].shape[:3]
    cs = [s_.shape[-1] for s_ in srcs] if src_c is None else list(src_c)
    kc = sum(pad_to(c, 64) for c in cs)
    dev = srcs[0].device
    for s_ in srcs:
        assert s_.dtype == torch.bfloat16 and s_.is_contiguous() and tuple(s_.shape[:3]) == (T, H, W)
    if out is None:
        out = torch.empty((T, H, W, kc), dtype=torch.uint8, device=dev)
    if s_a is None:
        s_a = torch.empty(T, dtype=torch.float32, device=dev)
    assert out.dtype == torch.uint8 and tuple(out.shape) == (T, H, W, kc) and out.is_contiguous()
    part = torch.empty(T * lib.QUANT_PARTS, dtype=torch.float32, device=dev)
    n = len(srcs)
    ptrs = (C.c_void_p * 3)(*([s_.data_ptr() for s_ in srcs] + [None] * (3 - n)))
    cc = (C.c_int32 * 3)(*(cs + [0] * (3 - n)))
    ld = (C.c_int32 * 3)(*([s_.shape[-1] for s_ in srcs] + [0] * (3 - n)))
    call('pf_quantize_e4m3_tiles', n, ptrs, cc, ld, T, H, W, part, out, s_a, stream_ptr())
    return out, s_a


def conv3_e4m3(pw, q, s_a, out, act=ACT_NONE, block_n=0):
    """The E4M3 halo conv: q / s_a from quantize_e4m3_tiles over sources with pw.src_c channels, pw from
    pack_weight_e4m3, out bf16 NHWC [T,H,W,ld]."""
    T, H, W, kc = q.shape
    assert q.dtype == torch.uint8 and kc == sum(pad_to(c, 64) for c in pw.src_c) and pw.taps == 9
    d = GemmDesc()
    d.num_src = len(pw.src_c)
    d.taps = 9
    d.a_mode = 1
    d.a_ptr[0] = q.data_ptr()
    for i, c in enumerate(pw.src_c):
        d.a_c[i], d.a_ld[i] = pad_to(c, 8), kc
    d.NB, d.H, d.W = T, H, W
    d.w_ptr = pw.w8.data_ptr()
    d.N, d.Ktot, d.block_n = pw.N, pw.Ktot, block_n
    d.bias = pw.bias.data_ptr() if pw.bias is not None else None
    d.act = act
    assert out.dtype == torch.bfloat16 and out.is_contiguous()
    d.out, d.out_ld = out.data_ptr(), out.shape[-1]
    d.a_e4m3, d.s_a, d.s_w = 1, s_a.data_ptr(), pw.w_scale.data_ptr()
    call('pf_gemm', C.byref(d), stream_ptr())
    return d


def e4m3_static_ratio(amax):
    """r = 448 / amax in fp32 (0 when amax == 0): the static quantize ratio of a calibrated amax (include/pf_b200.h)"""
    a = np.float32(amax)
    return float(np.float32(0.0) if a == 0 else np.float32(448.0) / a)


def e4m3_static_scale(amax):
    """amax / 448 in fp32: the dequantize scale of a calibrated amax"""
    return float(np.float32(amax) / np.float32(448.0))


def quantize_e4m3_static(srcs, amax, src_c=None, out=None):
    """srcs: bf16 NHWC maps [T,H,W,ld_i] (logical channels src_c[i], default the last dim) -> the e4m3 map [T,H,W,Kc]
    (uint8 storage, quantize_e4m3_tiles' layout) at the static ratio of `amax` (pf_quantize_e4m3_static, saturating)."""
    T, H, W = srcs[0].shape[:3]
    cs = [s_.shape[-1] for s_ in srcs] if src_c is None else list(src_c)
    kc = sum(pad_to(c, 64) for c in cs)
    for s_ in srcs:
        assert s_.dtype == torch.bfloat16 and s_.is_contiguous() and tuple(s_.shape[:3]) == (T, H, W)
    if out is None:
        out = torch.empty((T, H, W, kc), dtype=torch.uint8, device=srcs[0].device)
    assert out.dtype == torch.uint8 and tuple(out.shape) == (T, H, W, kc) and out.is_contiguous()
    n = len(srcs)
    ptrs = (C.c_void_p * 3)(*([s_.data_ptr() for s_ in srcs] + [None] * (3 - n)))
    cc = (C.c_int32 * 3)(*(cs + [0] * (3 - n)))
    ld = (C.c_int32 * 3)(*([s_.shape[-1] for s_ in srcs] + [0] * (3 - n)))
    call('pf_quantize_e4m3_static', n, ptrs, cc, ld, T, H, W, e4m3_static_ratio(amax), out, stream_ptr())
    return out


def conv3_e4m3_static(pw, q, amax, out, next_amax=None, act=ACT_RELU, block_n=0, res1=None, res2=None, copy=None,
                      copy_amax=None):
    """The static-scale E4M3 halo conv (pf_conv3_halo_e4m3_q8_kernel): q from quantize_e4m3_static at `amax`, pw from
    pack_weight_e4m3.  next_amax None: out bf16 NHWC [T,H,W,ld]; else out is the uint8 e4m3 map [T,H,W,ld >= pad64(N)]
    written at next_amax's ratio (the next conv's operand).
    res1 / res2 (bf16 NHWC [T,H,W,ld], added after the bias) and copy (the uint8 e4m3 map [T,H,W,ld >= pad64(N)] that
    receives the bf16 output's ReLU at copy_amax's ratio) run pf_conv3_halo_e4m3_res_kernel, with a bf16 out."""
    T, H, W, kc = q.shape
    assert q.dtype == torch.uint8 and kc == sum(pad_to(c, 64) for c in pw.src_c) and pw.taps == 9
    d = GemmDesc()
    d.num_src = len(pw.src_c)
    d.taps = 9
    d.a_mode = 1
    d.a_ptr[0] = q.data_ptr()
    for i, c in enumerate(pw.src_c):
        d.a_c[i], d.a_ld[i] = pad_to(c, 8), kc
    d.NB, d.H, d.W = T, H, W
    d.w_ptr = pw.w8.data_ptr()
    d.N, d.Ktot, d.block_n = pw.N, pw.Ktot, block_n
    d.bias = pw.bias.data_ptr() if pw.bias is not None else None
    d.act = act
    assert out.is_contiguous() and out.dtype == (torch.bfloat16 if next_amax is None else torch.uint8)
    d.out, d.out_ld = out.data_ptr(), out.shape[-1]
    d.a_e4m3, d.s_w = 1, pw.w_scale.data_ptr()
    d.a_static, d.a_scale = 1, e4m3_static_scale(amax)
    if next_amax is not None:
        d.out_e4m3, d.out_ratio = 1, e4m3_static_ratio(next_amax)
    for i, r in enumerate((res1, res2)):
        if r is not None:
            assert r.dtype == torch.bfloat16 and r.is_contiguous() and tuple(r.shape[:3]) == (T, H, W)
            setattr(d, 'res%d' % (i + 1), r.data_ptr())
            d.res_ld = r.shape[-1]
    if copy is not None:
        assert copy.dtype == torch.uint8 and copy.is_contiguous() and tuple(copy.shape[:3]) == (T, H, W)
        d.out2, d.out2_ld = copy.data_ptr(), copy.shape[-1]
        d.out2_e4m3, d.out2_ratio = 1, e4m3_static_ratio(copy_amax)
    call('pf_gemm', C.byref(d), stream_ptr())
    return d


def pack_weight_convT(weight, bias, k):
    """ConvTranspose2d(kernel == stride) weight [Cin, Cout, k, k]."""
    weight = weight.float().contiguous()
    cin, cout = weight.shape[0], weight.shape[1]
    cp = pad_to(cout, 32)
    dst = torch.empty((k * k * cp, pad_to(cin, 64)), dtype=torch.bfloat16, device=weight.device)
    call('pf_pack_weight_convT', weight, cin, cout, k, dst, stream_ptr())
    return PackedWeight(dst, bias.float().contiguous() if bias is not None else None, k * k * cp, [cin], 1, ps=k,
                        ps_cout=cout)


def gemm(pw, srcs, out, *, image=None, ps_image=None, M=None, act=ACT_NONE, res1=None, res2=None, gamma=None, out_col0=0, out2=None,
         vt=None, vt_col0=0, vt_seq=0, vt_seq_pad=0, src_c=None, block_n=0, tail=None, tail_out=None,
         skip_main=False, tile=None, resample=None):
    """srcs: list of bf16 tensors.  image=(NB,H,W) selects NHWC/conv addressing (srcs are [NB,H,W,ld]);
    otherwise srcs are [M, ld] matrices.  `out` may be bf16 or fp32; with `gamma` it is the fp32 residual stream
    updated in place (x += gamma * (acc + bias)).  resample[i] = True: source i is a [NB, h, w, ld] map of another size
    that the 3x3 conv reads through a fused bilinear (align_corners=True) resample to (H, W)."""
    d = GemmDesc()
    d.num_src = len(srcs)
    d.taps = pw.taps
    cs = pw.src_c if src_c is None else src_c
    assert len(cs) == len(srcs)
    for i, s in enumerate(srcs):
        assert s.dtype == torch.bfloat16 and s.is_contiguous()
        d.a_ptr[i] = s.data_ptr()
        d.a_c[i] = pad_to(cs[i], 8)
        d.a_ld[i] = s.shape[-1]
        assert d.a_c[i] <= s.shape[-1]
        if resample is not None and resample[i]:
            d.rs_h[i], d.rs_w[i] = s.shape[1], s.shape[2]
    if image is not None:
        d.a_mode = 1
        d.NB, d.H, d.W = image
        rows = d.NB * d.H * d.W
        if tile is not None:        # pin the pixel tile (bh, bw): selects the per-tap TMA kernel for 3x3 convs
            d.bh, d.bw = tile
    else:
        d.a_mode = 0
        d.M = M if M is not None else srcs[0].shape[0]
        rows = d.M
        if pw.ps > 1:
            d.NB, d.H, d.W = ps_image
    d.w_ptr = pw.w.data_ptr()
    d.N = pw.N
    d.Ktot = pw.Ktot
    d.block_n = block_n
    d.bias = pw.bias.data_ptr() if pw.bias is not None else None
    d.act = act
    if res1 is not None:
        d.res1 = res1.data_ptr()
        d.res_ld = res1.shape[-1]
    if res2 is not None:
        d.res2 = res2.data_ptr()
        assert res2.shape[-1] == d.res_ld
    if gamma is not None:
        assert out.dtype == torch.float32
        d.gamma = gamma.data_ptr()
    d.out = out.data_ptr()
    d.out_f32 = 1 if out.dtype == torch.float32 else 0
    d.out_ld = out.shape[-1]
    d.out_col0 = out_col0
    if out2 is not None:
        d.out2 = out2.data_ptr()
        d.out2_ld = out2.shape[-1]
    d.ps, d.ps_cout = pw.ps, pw.ps_cout
    if vt is not None:
        d.vt = vt.data_ptr()
        d.vt_col0, d.vt_seq, d.vt_seq_pad, d.vt_dim = vt_col0, vt_seq, vt_seq_pad, pw.N - vt_col0
    if tail is not None:
        # fused trailing 1x1 layer: tail = (w2 fp32 [n2, N], b2 fp32 [n2] or None, act2)
        w2, b2, act2 = tail
        assert w2.dtype == torch.float32 and w2.is_contiguous() and w2.shape[1] == pw.N and tail_out.dtype == torch.float32
        d.w2, d.b2 = w2.data_ptr(), (b2.data_ptr() if b2 is not None else None)
        d.n2, d.act2, d.skip_main = w2.shape[0], act2, 1 if skip_main else 0
        d.out3, d.out3_ld = tail_out.data_ptr(), tail_out.shape[-1]
    call('pf_gemm', C.byref(d), stream_ptr())
    return d


def linear_e4m3(pw, q, amax, out, act=ACT_NONE, out_f32=False, gamma=None, vt=None, out_amax=None, block_n=0):
    """The E4M3 ping-pong GEMM (pf_gemm_pp_e4m3_kernel) over q, an e4m3 matrix [M, K] (uint8 storage) quantized at the
    static ratio of `amax`, with pw from pack_weight_e4m3.  out: bf16 [M, ld] (vt = (buffer [B*D_v, seq_pad], vt_col0,
    seq): the fused qkv projection's V^T third), fp32 [M, ld] (gamma: out += gamma * v), or, with out_amax, the e4m3
    matrix [M, ld bytes] of the next linear at that amax's ratio."""
    M, K = q.shape
    assert q.dtype == torch.uint8 and pw.taps == 1 and pw.Ktot == K
    d = GemmDesc()
    d.num_src, d.taps, d.a_mode = 1, 1, 0
    d.a_ptr[0], d.a_c[0], d.a_ld[0] = q.data_ptr(), K, q.stride(0)
    d.M = M
    d.w_ptr = pw.w8.data_ptr()
    d.N, d.Ktot, d.block_n = pw.N, pw.Ktot, block_n
    d.bias = pw.bias.data_ptr() if pw.bias is not None else None
    d.act = act
    d.out, d.out_ld = out.data_ptr(), out.stride(0)
    d.out_f32 = 1 if out_f32 or gamma is not None else 0
    d.gamma = gamma.data_ptr() if gamma is not None else None
    if vt is not None:
        vbuf, d.vt_col0, d.vt_seq = vt
        d.vt, d.vt_seq_pad, d.vt_dim = vbuf.data_ptr(), vbuf.shape[-1], pw.N - d.vt_col0
    d.a_e4m3, d.a_static, d.a_scale, d.s_w = 1, 1, e4m3_static_scale(amax), pw.w_scale.data_ptr()
    if out_amax is not None:
        d.out_e4m3, d.out_ratio = 1, e4m3_static_ratio(out_amax)
    call('pf_gemm', C.byref(d), stream_ptr())
    return d


def layernorm_e4m3(x, w, b, eps, amax, out):
    """pf_layernorm_e4m3: LayerNorm of fp32 x [rows, ld] into the e4m3 matrix out [rows, ld bytes] at amax's ratio"""
    call('pf_layernorm_e4m3', x, x.stride(0), w, b, C.c_float(eps), x.shape[0], w.shape[0], C.c_float(e4m3_static_ratio(amax)),
         out, out.stride(0), stream_ptr())


def gemm_convT(pw, src, image, out):
    """ConvTranspose k==s: src [NB*H*W, ld] rows in (n,y,x) order, out NHWC [NB, H*k, W*k, ld_out]."""
    return gemm(pw, [src], out, ps_image=image, M=image[0] * image[1] * image[2])


def layernorm(x, w, b, eps, out, rows=None, C_=None):
    rows = x.shape[0] if rows is None else rows
    C_ = w.shape[0] if C_ is None else C_
    call('pf_layernorm', x, x.shape[-1], w, b, C.c_float(eps), rows, C_, out, out.shape[-1], stream_ptr())


def attention(qk, vt, B, seq, seq_pad, heads, scale, out):
    call('pf_attention', qk, qk.shape[-1], vt, B, seq, seq_pad, heads, C.c_float(scale), out, out.shape[-1],
         stream_ptr())


def resize_bilinear(x, C_, OH, OW, out, out_col0=0):
    B, H, W, ld = x.shape
    call('pf_resize_bilinear', x, B, H, W, pad_to(C_, 8), ld, OH, OW, out, out.shape[-1], out_col0, stream_ptr())


def roi_crop_zoom(feat, C_, boxes, scale, out, out_col0=0, tile_image=None):
    """feat [B,h,w,ld] bf16 or [B,h,w] / [h,w] fp32 (depth); boxes [T,4] fp32 device; tile_image: int32 [T] device
    tensor, the image of `feat` each box reads (None: image 0)."""
    T = boxes.shape[0]
    if feat.dtype == torch.float32:
        h, w = feat.shape[-2:]
        call('pf_roi_crop_zoom_batched', feat, 1, h, w, 1, 1, tile_image, boxes, T, C.c_float(scale), out, 1, 0,
             stream_ptr())
    else:
        _, h, w, ld = feat.shape
        call('pf_roi_crop_zoom_batched', feat, 0, h, w, pad_to(C_, 8), ld, tile_image, boxes, T, C.c_float(scale), out,
             out.shape[-1], out_col0, stream_ptr())


def crop_resize(img, origins, tile_image, th, tw, ph, pw, out):
    """Tiles of img [B,3,H,W] (or [3,H,W]) fp32: tile t = image tile_image[t] (None: image 0) at origins[t] (int32
    [T,2] device, y, x), th x tw pixels, resized to out [T,3,ph,pw] (bilinear, align_corners=True)."""
    H, W = img.shape[-2:]
    call('pf_crop_resize_batched', img, H, W, origins, tile_image, origins.shape[0], th, tw, ph, pw, out, stream_ptr())


def crop_table(images, sizes, out):
    """Write the pf_crop_resize_multi descriptors of `images` (each a contiguous fp32 [1,3,H,W] or [3,H,W] device
    tensor) with tiles of sizes[b] = (th, tw) into `out`, a uint8 device tensor of len(images) descriptors."""
    arr = (lib.CropImage * len(images))()
    for d, img, (th, tw) in zip(arr, images, sizes):
        assert img.dtype == torch.float32 and img.is_cuda and img.is_contiguous() and img.shape[-3] == 3
        assert 0 < th <= img.shape[-2] and 0 < tw <= img.shape[-1]
        d.img, (d.H, d.W), d.th, d.tw = img.data_ptr(), img.shape[-2:], th, tw
    assert out.dtype == torch.uint8 and out.numel() == C.sizeof(arr)
    out.copy_(torch.frombuffer(bytearray(arr), dtype=torch.uint8))
    return out


def crop_table_bytes(n):
    return n * C.sizeof(lib.CropImage)


def crop_resize_multi(table, origins, tile_image, ph, pw, out):
    """Tiles of images of different sizes: tile t is a crop of the image of descriptor tile_image[t] of `table`
    (crop_table) at origins[t] (int32 [T,2] device, y, x), resized to out [T,3,ph,pw] (bilinear, align_corners=True)."""
    call('pf_crop_resize_multi', table, origins, tile_image, origins.shape[0], ph, pw, out, stream_ptr())


def maxpool2(x, C_, out):
    B, H, W, ld = x.shape
    call('pf_maxpool2', x, B, H, W, pad_to(C_, 8), ld, out, out.shape[-1], stream_ptr())


def seed_bins(S, nbins, flags, min_depth, max_depth, out):
    """pf_seed_bins: the seed regressor's fp32 `_net` output S [..., S_ld] (one row per pixel) -> bin centres
    out [..., nbins].  flags: lib.SEED_NORMED (SeedBinRegressor) | lib.SEED_TO_UNIT ((c - min) / (max - min))."""
    call('pf_seed_bins', S, S.shape[-1], S.numel() // S.shape[-1], nbins, flags, C.c_float(min_depth),
         C.c_float(max_depth), out, stream_ptr())


def attractor_normed(A, nA, b_prev, flags, min_depth, max_depth, b_out, centers=None):
    """pf_attractor_normed: A fp32 [B, H, W, A_ld] (the even `_net` channels, ReLU'd), b_prev [B, h, w, nbins] ->
    b_out [B, H, W, nbins] and, when given, the sorted and clipped metric centres [B, H, W, nbins]."""
    B, H, W, A_ld = A.shape
    _, PH, PW, nb = b_prev.shape
    call('pf_attractor_normed', A, A_ld, nA, b_prev, PH, PW, B, H, W, nb, flags, C.c_float(min_depth),
         C.c_float(max_depth), b_out, centers, stream_ptr())


def depth_to_points(depth, inv_f, rt, image, points, colors=None):
    """pf_depth_to_points: depth [.., H, W] fp32 -> points [H*W, 3] fp32; rt: 12 floats (R row-major, then t) or None
    (identity, zero); image: planar RGB [.., 3, H, W] fp32 or None, whose colours go to colors [H*W, 3] uint8."""
    H, W = depth.shape[-2:]
    rt_c = None if rt is None else (C.c_float * 12)(*rt)
    call('pf_depth_to_points', depth, H, W, C.c_float(inv_f), rt_c, image, points, colors, stream_ptr())


def depth_edge_mask(depth, threshold, out):
    """pf_depth_edge_mask: depth [.., H, W] fp32 -> out [H, W] (uint8 or bool storage), 1 where the vertex is kept."""
    H, W = depth.shape[-2:]
    call('pf_depth_edge_mask', depth, H, W, C.c_float(threshold), out, stream_ptr())


def mesh_scan_blocks(h, w):
    """blocks of pf_mesh_quad_counts' scan: `offsets` holds this many int64 offsets plus the total"""
    return ((h - 1) * (w - 1) + lib.MESH_SCAN_BLOCK - 1) // lib.MESH_SCAN_BLOCK


def mesh_quad_counts(mask, h, w, flags, offsets):
    """pf_mesh_quad_counts: vertex mask [h, w] (uint8 / bool) -> kept-triangle flags [(h-1)(w-1)] uint8 and
    offsets [mesh_scan_blocks(h, w) + 1] int64 (per-block output offsets, then the triangle count)."""
    call('pf_mesh_quad_counts', mask, h, w, flags, offsets, stream_ptr())


def mesh_triangles(flags, offsets, h, w, faces):
    """pf_mesh_triangles: the kept triangles into faces [n, 3] int32 (flags None: all 2 (h-1)(w-1) of them); writes
    nothing past faces.shape[0] rows."""
    call('pf_mesh_triangles', flags, offsets, h, w, faces, C.c_int64(faces.shape[0]), stream_ptr())


def ply_pack_vertices(points, colors, out):
    """pf_ply_pack_vertices: points [n, 3] fp32 + colors [n, 3] uint8 -> out [15 n] uint8 PLY vertex records"""
    call('pf_ply_pack_vertices', points, colors, C.c_int64(points.shape[0]), out, stream_ptr())


def ply_pack_faces(faces, out):
    """pf_ply_pack_faces: faces [n, 3] int32 -> out [13 n] uint8 PLY face records"""
    call('pf_ply_pack_faces', faces, C.c_int64(faces.shape[0]), out, stream_ptr())
