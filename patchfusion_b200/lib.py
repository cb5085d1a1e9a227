"""ctypes binding of libpf_b200.so (C ABI declared in include/pf_b200.h).

There is no CPU or PyTorch fallback: if the shared library has not been built (`python -m patchfusion_b200.build`
or `__graft_entry__.build()`), loading raises, and every entry point raises `PFError` on a non-zero status.
torch is used only to own device memory and the CUDA stream.
"""
import ctypes as C
import os

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, os.environ.get('PF_B200_LIBNAME', 'libpf_b200.so'))

ACT_NONE, ACT_RELU, ACT_GELU, ACT_SOFTPLUS = 0, 1, 2, 3
OPT_TMA_EPILOGUE, OPT_HALO_MULTICAST, OPT_GEMM_MULTICAST, OPT_FUSED_RESAMPLE, OPT_PDL, OPT_RESIZE_SEPARABLE = 0, 1, 2, 3, 4, 5


class PFError(RuntimeError):
    pass


class GemmDesc(C.Structure):
    """Mirror of `pf_gemm_desc` (include/pf_b200.h)."""
    _fields_ = [
        ('num_src', C.c_int32), ('a_mode', C.c_int32), ('taps', C.c_int32), ('chunks', C.c_int32 * 3),
        ('a_ptr', C.c_void_p * 3), ('a_c', C.c_int32 * 3), ('a_ld', C.c_int32 * 3),
        ('M', C.c_int32), ('NB', C.c_int32), ('H', C.c_int32), ('W', C.c_int32), ('bh', C.c_int32), ('bw', C.c_int32),
        ('tiles_y', C.c_int32), ('tiles_x', C.c_int32), ('m_tiles', C.c_int32),
        ('w_ptr', C.c_void_p), ('N', C.c_int32), ('Ktot', C.c_int32), ('block_n', C.c_int32), ('n_tiles', C.c_int32),
        ('bias', C.c_void_p), ('act', C.c_int32),
        ('res1', C.c_void_p), ('res2', C.c_void_p), ('res_ld', C.c_int32),
        ('gamma', C.c_void_p),
        ('out', C.c_void_p), ('out_f32', C.c_int32), ('out_ld', C.c_int32), ('out_col0', C.c_int32),
        ('out2', C.c_void_p), ('out2_ld', C.c_int32),
        ('ps', C.c_int32), ('ps_cout', C.c_int32),
        ('vt', C.c_void_p), ('vt_col0', C.c_int32), ('vt_seq', C.c_int32), ('vt_seq_pad', C.c_int32),
        ('vt_dim', C.c_int32),
        ('w2', C.c_void_p), ('b2', C.c_void_p), ('n2', C.c_int32), ('act2', C.c_int32), ('skip_main', C.c_int32),
        ('out3', C.c_void_p), ('out3_ld', C.c_int32),
        ('rs_h', C.c_int32 * 3), ('rs_w', C.c_int32 * 3),
    ]


class CropImage(C.Structure):
    """Mirror of `pf_crop_image` (include/pf_b200.h): one image of a pf_crop_resize_multi table."""
    _fields_ = [('img', C.c_void_p), ('H', C.c_int32), ('W', C.c_int32), ('th', C.c_int32), ('tw', C.c_int32)]


_i, _f, _p, _ll = C.c_int32, C.c_float, C.c_void_p, C.c_int64
# name -> argument types (all return int status), in the order of include/pf_b200.h
SIGNATURES = {
    'pf_set_option': [_i, _i],
    'pf_profile_start': [_p],
    'pf_profile_stop': [],
    'pf_profile_get': [_i, _p, _p, _p, _p],
    'pf_gemm_timeline': [_p, _i],
    'pf_gemm': [C.POINTER(GemmDesc), _p],
    'pf_pack_weight': [_p, _i, _i, _i, C.POINTER(C.c_int32), _i, _p, _p, _p],
    'pf_pack_weight_convT': [_p, _i, _i, _i, _p, _p],
    'pf_layernorm': [_p, _i, _p, _p, _f, _i, _i, _p, _i, _p],
    'pf_layernorm_grouped': [_p, _i, _p, _p, _f, _i, _i, _i, _i, _i, _p, _i, _p],
    'pf_attention': [_p, _i, _p, _i, _i, _i, _i, _f, _p, _i, _p],
    'pf_patch_im2col': [_p, _i, _i, _i, _p, _i, _p],
    'pf_assemble_tokens': [_p, _p, _p, _i, _i, _i, _p, _p],
    'pf_resize_bilinear': [_p, _i, _i, _i, _i, _i, _i, _i, _p, _i, _i, _p],
    'pf_resize_bilinear_f32': [_p, _i, _i, _i, _i, _i, _i, _p, _p],
    'pf_roi_crop_zoom': [_p, _i, _i, _i, _i, _i, _p, _i, _f, _p, _i, _i, _p],
    'pf_roi_crop_zoom_batched': [_p, _i, _i, _i, _i, _i, _p, _p, _i, _f, _p, _i, _i, _p],
    'pf_maxpool2': [_p, _i, _i, _i, _i, _i, _p, _i, _p],
    'pf_im2col_3x3_s2': [_p, _i, _i, _i, _i, _i, _p, _p],
    'pf_crop_resize': [_p, _i, _i, _p, _i, _i, _i, _i, _i, _p, _p],
    'pf_crop_resize_batched': [_p, _i, _i, _p, _p, _i, _i, _i, _i, _i, _p, _p],
    'pf_crop_resize_multi': [_p, _p, _p, _i, _i, _i, _p, _p],
    'pf_pack_unet_input': [_p, _p, _p, _i, _i, _i, _p, _i, _p],
    'pf_f32_to_bf16': [_p, _ll, _p, _p],
    'pf_ingest_u8': [_p, _i, _i, _i, _i, _i, _p, _p],
    'pf_depth_to_u16': [_p, _i, _i, _i, _i, _f, _p, _p],
    'pf_ingest_raw_u8': [_p, _i, _i, _i, _p, _p],
    'pf_gt_prepare': [_p, _i, _i, _i, _f, _f, _f, _p, _p, _p],
    'pf_depth_metrics': [_p, _i, _i, _p, _i, _i, _f, _f, _p, _p, _p, _i, _p, _p],
    'pf_colorize_u8': [_p, _ll, _f, _f, _f, _p, _i, _p, _p],
    'pf_g2l_embed': [_p, _i, _p, _i, _i, _p, _p],
    'pf_swin_norm_pad': [_p, _p, _p, _f, _i, _i, _i, _i, _i, _p, _p],
    'pf_window_attention': [_p, _p, _i, _i, _i, _i, _i, _p, _p],
    'pf_swin_residual_crop': [_p, _p, _i, _i, _i, _i, _p],
    'pf_g2l_embed_batched': [_p, _i, _p, _i, _i, _i, _p, _p],
    'pf_swin_norm_pad_batched': [_p, _p, _p, _f, _i, _i, _i, _i, _i, _i, _p, _p],
    'pf_window_attention_batched': [_p, _p, _i, _i, _i, _i, _i, _i, _p, _p],
    'pf_swin_residual_crop_batched': [_p, _p, _i, _i, _i, _i, _i, _i, _p],
    'pf_add_upsampled': [_p, _i, _i, _i, _i, _p, _i, _i, _p, _p],
    'pf_attractor': [_p, _i, _i, _p, _i, _i, _i, _i, _i, _i, _i, _p, _p],
    'pf_logbinom_depth': [_p, _i, _p, _i, _i, _i, _i, _i, _i, _f, _f, _p, _p],
    'pf_stitch_accumulate': [_p, _p, _i, _i, _p, _i, _i, _i, _p, _p, _i, _i, _p],
    'pf_stitch_gather': [_p, _p, _i, _i, _i, _p, _i, _i, _p, _p, _i, _i, _p, _p, _p, _p],
    'pf_stitch_finalize': [_p, _p, _ll, _p, _p],
    'pf_stitch_reduce': [_p, _i, _ll, _p],
    'pf_stitch_resize': [_p, _p, _i, _i, _i, _i, _p, _p, _p],
}
EXPORTS = sorted(list(SIGNATURES) + ['pf_last_error', 'pf_version', 'pf_launch_count', 'pf_branch_workspace_bytes', 'pf_branch_forward',
                  'pf_g2l_workspace_bytes', 'pf_g2l_forward', 'pf_fusion_workspace_bytes', 'pf_fusion_forward',
                  'pf_fusion_forward_batched'])

_lib = None


def load():
    """Load the CUDA library; raises if it has not been built (no fallback path exists)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise PFError('%s is missing: build it with `python -m patchfusion_b200.build` '
                          '(the hot path has no CPU/PyTorch fallback)' % LIB_PATH)
        lib = C.CDLL(LIB_PATH)
        for name, args in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.argtypes = args
            fn.restype = C.c_int
        lib.pf_last_error.restype = C.c_char_p
        lib.pf_version.restype = C.c_int
        lib.pf_launch_count.restype = C.c_longlong
        _lib = lib
    return _lib


def launch_count():
    return int(load().pf_launch_count())


def stream_ptr():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    if t is None:
        return None
    if isinstance(t, int):
        return t
    assert t.is_cuda, 'libpf_b200 takes device pointers only'
    return t.data_ptr()


class Profiler:
    """Per-launch CUDA-event timing inside the library (pf_profile_start/stop/get; bench.py's roofline pass): every
    kernel libpf_b200 launches on the current stream between start() and stop() is recorded with its name, shape
    label, algorithmic flops and duration.  While `lib.PROFILER` is set the model runs eagerly on one stream."""

    def __init__(self):
        self.records = []          # (kernel name, label, flops, ms)

    def start(self):
        load().pf_profile_start(stream_ptr())

    def stop(self):
        h = load()
        h.pf_profile_get.argtypes = [C.c_int32, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), C.POINTER(C.c_double),
                                     C.POINTER(C.c_float)]
        n = h.pf_profile_stop()
        name, label, fl, ms = C.c_char_p(), C.c_char_p(), C.c_double(), C.c_float()
        for i in range(n):
            if h.pf_profile_get(i, C.byref(name), C.byref(label), C.byref(fl), C.byref(ms)) != 0:
                raise PFError(h.pf_last_error().decode())
            self.records.append((name.value.decode(), label.value.decode(), fl.value, ms.value))
        return self.records


PROFILER = None


def call(name, *args):
    _call(name, *args)


def _call(name, *args):
    lib = load()
    conv = []
    for a in args:
        if isinstance(a, torch.Tensor):
            if not a.is_contiguous():
                raise PFError('%s: non-contiguous tensor passed as a raw pointer' % name)
            conv.append(C.c_void_p(ptr(a)))
        elif a is None:
            conv.append(None)
        else:
            conv.append(a)
    st = getattr(lib, name)(*conv)
    if st != 0:
        raise PFError('%s failed: %s' % (name, lib.pf_last_error().decode()))
