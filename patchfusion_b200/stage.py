"""ctypes mirrors of the stage-level C ABI (include/pf_b200.h: pf_layer ... pf_fusion, pf_map, pf_branch_out) and the
calls `pf_branch_forward` / `pf_g2l_forward` / `pf_fusion_forward`.  tests/test_cabi.py checks every struct's size and
field offsets against the header with gcc."""
import ctypes as C

import torch

from . import lib

i32, f32, vp = C.c_int32, C.c_float, C.c_void_p


class PfLayer(C.Structure):
    _fields_ = [('w', vp), ('bias', vp), ('N', i32), ('Ktot', i32), ('taps', i32), ('num_src', i32), ('src_c', i32 * 3),
                ('ps', i32), ('ps_cout', i32), ('w2', vp), ('b2', vp), ('n2', i32), ('w8', vp), ('w_scale', vp),
                ('a_amax', vp)]


class PfVitBlock(C.Structure):
    _fields_ = [('n1w', vp), ('n1b', vp), ('n2w', vp), ('n2b', vp), ('ls1', vp), ('ls2', vp),
                ('qkv', PfLayer), ('proj', PfLayer), ('fc1', PfLayer), ('fc2', PfLayer)]


class PfHead(C.Structure):
    _fields_ = [('seed0', PfLayer), ('seed2', PfLayer), ('seedproj0', PfLayer), ('seedproj2', PfLayer),
                ('proj0', PfLayer * 4), ('proj2', PfLayer * 4), ('att0', PfLayer * 4), ('att2', PfLayer * 4),
                ('clb0', PfLayer), ('n_attractors', i32 * 4), ('n_bins', i32), ('bin_embedding_dim', i32),
                ('attractor_flags', i32), ('has_rel', i32), ('min_temp', f32), ('max_temp', f32),
                ('bin_centers_type', i32), ('min_depth', f32), ('max_depth', f32)]


class PfBranch(C.Structure):
    _fields_ = [('H', i32), ('W', i32), ('dim', i32), ('depth', i32), ('heads', i32), ('features', i32),
                ('out_channels', i32 * 4), ('patch', PfLayer), ('pos', vp), ('cls', vp), ('blocks', C.POINTER(PfVitBlock)),
                ('nw', vp), ('nb', vp), ('proj', PfLayer * 4), ('rs0', PfLayer), ('rs1', PfLayer), ('rs3', PfLayer),
                ('rn', PfLayer * 4), ('ff_out', PfLayer * 4), ('ff_c1', (PfLayer * 2) * 4), ('ff_c2', (PfLayer * 2) * 4),
                ('oc1', PfLayer), ('oc2', PfLayer), ('conv2', PfLayer), ('head', PfHead)]


class PfG2LBlock(C.Structure):
    _fields_ = [('n1w', vp), ('n1b', vp), ('n2w', vp), ('n2b', vp), ('table', vp),
                ('qkv', PfLayer), ('proj', PfLayer), ('fc1', PfLayer), ('fc2', PfLayer)]


class PfG2LLevel(C.Structure):
    _fields_ = [('C', i32), ('heads', i32), ('depth', i32), ('ape', vp), ('ape_rows', i32), ('nw', vp), ('nb', vp),
                ('ones', vp), ('blocks', C.POINTER(PfG2LBlock))]


class PfFusion(C.Structure):
    _fields_ = [('H', i32), ('W', i32), ('fc', PfLayer * 5), ('inc', PfLayer * 2), ('down', (PfLayer * 2) * 5),
                ('up', (PfLayer * 2) * 5), ('cv', (PfLayer * 2) * 6), ('g2l', PfG2LLevel * 6), ('head', PfHead)]


class PfMap(C.Structure):
    _fields_ = [('ptr', vp), ('B', i32), ('H', i32), ('W', i32), ('C', i32), ('ld', i32)]


class PfBranchOut(C.Structure):
    _fields_ = [('depth', vp), ('feats', PfMap * 6)]


TAP_FN = C.CFUNCTYPE(None, vp, C.c_char_p, vp, i32, C.c_int64, i32, i32)
STRUCTS = {'pf_layer': PfLayer, 'pf_vit_block': PfVitBlock, 'pf_head': PfHead, 'pf_branch': PfBranch,
           'pf_g2l_block': PfG2LBlock, 'pf_g2l_level': PfG2LLevel, 'pf_fusion': PfFusion, 'pf_map': PfMap,
           'pf_branch_out': PfBranchOut}

_bound = False


def _bind():
    global _bound
    if _bound:
        return lib.load()
    h = lib.load()
    h.pf_branch_workspace_bytes.restype = C.c_size_t
    h.pf_branch_workspace_bytes.argtypes = [C.POINTER(PfBranch), i32]
    h.pf_g2l_workspace_bytes.restype = C.c_size_t
    h.pf_g2l_workspace_bytes.argtypes = [C.POINTER(PfFusion), C.POINTER(PfMap)]
    h.pf_fusion_workspace_bytes.restype = C.c_size_t
    h.pf_fusion_workspace_bytes.argtypes = [C.POINTER(PfFusion), i32, C.POINTER(PfMap)]
    h.pf_branch_forward.restype = C.c_int
    h.pf_branch_forward.argtypes = [C.POINTER(PfBranch), vp, i32, vp, C.c_size_t, C.POINTER(PfBranchOut), vp, vp, vp]
    h.pf_g2l_forward.restype = C.c_int
    h.pf_g2l_forward.argtypes = [C.POINTER(PfFusion), C.POINTER(PfMap), vp, C.c_size_t, C.POINTER(PfMap), vp, vp, vp]
    h.pf_fusion_forward.restype = C.c_int
    h.pf_fusion_forward.argtypes = [C.POINTER(PfFusion), vp, vp, i32, vp, C.POINTER(PfMap), vp, C.POINTER(PfMap),
                                    C.POINTER(PfMap), vp, C.c_size_t, vp, vp, vp, vp]
    h.pf_fusion_forward_batched.restype = C.c_int
    h.pf_fusion_forward_batched.argtypes = [C.POINTER(PfFusion), vp, vp, vp, i32, vp, C.POINTER(PfMap), vp,
                                            C.POINTER(PfMap), C.POINTER(PfMap), vp, C.c_size_t, vp, vp, vp, vp]
    _bound = True
    return h


STAGE_EXPORTS = ['pf_branch_workspace_bytes', 'pf_branch_forward', 'pf_g2l_workspace_bytes', 'pf_g2l_forward',
                 'pf_fusion_workspace_bytes', 'pf_fusion_forward', 'pf_fusion_forward_batched']


def _check(rc, what):
    if rc != 0:
        raise lib.PFError('%s failed: %s' % (what, lib.load().pf_last_error().decode()))


def layer(pw, tail=None):
    """PackedWeight (+ optional fp32 trailing layer (w2 [n2, N], b2)) -> PfLayer.  The caller keeps the tensors alive.
    An FP8 layer (PackedWeight.w8 set) carries its e4m3 panel and scales, and its bf16 panel only when it has one."""
    L = PfLayer()
    L.w = pw.w.data_ptr() if pw.w is not None else None
    if getattr(pw, 'w8', None) is not None:
        L.w8, L.w_scale = pw.w8.data_ptr(), pw.w_scale.data_ptr()
    L.bias = pw.bias.data_ptr() if pw.bias is not None else None
    L.N, L.Ktot, L.taps = pw.N, pw.Ktot, pw.taps
    L.num_src = len(pw.src_c)
    for i, c in enumerate(pw.src_c):
        L.src_c[i] = c
    L.ps = pw.ps if pw.ps > 1 else 0
    L.ps_cout = pw.ps_cout
    if tail is not None:
        w2, b2 = tail
        assert w2.dtype == torch.float32 and w2.is_contiguous() and w2.shape[1] == pw.N and w2.shape[0] <= 16
        L.w2, L.b2, L.n2 = w2.data_ptr(), (b2.data_ptr() if b2 is not None else None), w2.shape[0]
    return L


def branch_workspace_bytes(cb, B):
    return int(_bind().pf_branch_workspace_bytes(C.byref(cb), B))


def g2l_workspace_bytes(cf, maps):
    return int(_bind().pf_g2l_workspace_bytes(C.byref(cf), maps))


def fusion_workspace_bytes(cf, T, maps):
    return int(_bind().pf_fusion_workspace_bytes(C.byref(cf), T, maps))


def count_stage_launches(fn):
    return fn()


def branch_forward(cb, images, B, ws_ptr, ws_bytes, tap=None):
    out = PfBranchOut()
    cbk = TAP_FN(tap) if tap is not None else None
    rc = _bind().pf_branch_forward(C.byref(cb), images.data_ptr(), B, ws_ptr, ws_bytes, C.byref(out),
                                   C.cast(cbk, vp) if cbk is not None else None, None, lib.stream_ptr())
    _check(rc, 'pf_branch_forward')
    return out


def g2l_forward(cf, maps, ws_ptr, ws_bytes, tap=None):
    out = (PfMap * 6)()
    cbk = TAP_FN(tap) if tap is not None else None
    rc = _bind().pf_g2l_forward(C.byref(cf), maps, ws_ptr, ws_bytes, out, C.cast(cbk, vp) if cbk is not None else None,
                                None, lib.stream_ptr())
    _check(rc, 'pf_g2l_forward')
    return out


def fusion_forward(cf, crops, boxes, T, fine_depth, fine_maps, coarse_depth, coarse_maps, g2l_maps, ws_ptr, ws_bytes,
                   depth_out, tap=None, tile_image=None):
    """tile_image (int32 [T] device tensor or None): the image of the batch-B coarse inputs each tile reads."""
    cbk = TAP_FN(tap) if tap is not None else None
    ti = tile_image.data_ptr() if tile_image is not None else None
    rc = _bind().pf_fusion_forward_batched(C.byref(cf), crops.data_ptr(), boxes.data_ptr(), ti, T, fine_depth.data_ptr(),
                                           fine_maps, coarse_depth.data_ptr(), coarse_maps, g2l_maps, ws_ptr, ws_bytes,
                                           depth_out.data_ptr(), C.cast(cbk, vp) if cbk is not None else None, None,
                                           lib.stream_ptr())
    _check(rc, 'pf_fusion_forward')
