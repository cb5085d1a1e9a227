"""GPU versions of the two callers either side of the hot path (SURVEY.md §8f): image ingest
(`estimator/datasets/general_dataset.py:22-47,188-219`) and the uint16 depth writer
(`estimator/tester/tester.py:66-76`, `tools/test_single_forward.py:26`)."""
import ctypes as C

import numpy as np
import torch

from . import ops


def ingest(image_u8, image_raw_shape, device, bgr=True):
    """image_u8: HxWx3 uint8 (numpy array as returned by cv2.imread, or a torch tensor).  Returns image_hr
    (1,3,H',W') fp32 in [0,1] on `device`, bicubic-resized (align_corners=True) to image_raw_shape."""
    if isinstance(image_u8, np.ndarray):
        image_u8 = torch.from_numpy(np.ascontiguousarray(image_u8))
    assert image_u8.dtype == torch.uint8 and image_u8.dim() == 3 and image_u8.shape[2] == 3
    src = image_u8.to(device, non_blocking=True).contiguous()
    H, W = src.shape[:2]
    OH, OW = image_raw_shape
    out = torch.empty((1, 3, OH, OW), dtype=torch.float32, device=device)
    ops.call('pf_ingest_u8', src, H, W, 1 if bgr else 0, OH, OW, out, ops.stream_ptr())
    return out


def ingest_raw(image_u8, bgr=True):
    """image_u8: HxWx3 uint8 tensor on the GPU (a U4K raw frame, stored BGR).  Returns image_hr (1,3,H,W) fp32 RGB,
    u8 / 255 correctly rounded at the same size (`u4k_dataset.py:126-129`; no resample)."""
    assert image_u8.is_cuda and image_u8.dtype == torch.uint8 and image_u8.dim() == 3 and image_u8.shape[2] == 3
    src = image_u8.contiguous()
    H, W = src.shape[:2]
    out = torch.empty((1, 3, H, W), dtype=torch.float32, device=src.device)
    ops.call('pf_ingest_raw_u8', src, H, W, 1 if bgr else 0, out, ops.stream_ptr())
    return out


GT_KINDS = {'u4k': 0, 'mid': 1, 'eth3d': 2, 'cityscapes': 3}
GT_SOURCE_DTYPES = {'u4k': torch.float32, 'mid': torch.float32, 'eth3d': torch.float32, 'cityscapes': torch.uint16}


def gt_prepare(src, kind, factor=0.0, doffs=0.0, th=1.0):
    """Ground truth of one evaluation image on the GPU (pf_gt_prepare): src [H,W] on the device (fp32; uint16 for
    'cityscapes') -> (depth_gt (1,1,H,W) fp32, boundary (1,1,H,W) uint8), bit-identical to the reference's numpy
    branch of that dataset.  factor / doffs are the reference's Python floats; they are rounded to float32 here, as
    numpy 2 does when it combines them with a float32 array."""
    if kind not in GT_KINDS:
        raise NotImplementedError('ground truth of kind %r' % (kind,))
    assert src.is_cuda and src.dim() == 2 and src.dtype == GT_SOURCE_DTYPES[kind], (src.dtype, kind)
    src = src.contiguous()
    H, W = src.shape
    depth = torch.empty((1, 1, H, W), dtype=torch.float32, device=src.device)
    boundary = torch.empty((1, 1, H, W), dtype=torch.uint8, device=src.device)
    ops.call('pf_gt_prepare', src, GT_KINDS[kind], H, W, C.c_float(factor), C.c_float(doffs), C.c_float(th), depth,
             boundary, ops.stream_ptr())
    return depth, boundary


def depth_to_u16(depth, size=None, scale=256.0):
    """depth (1,1,h,w) or (h,w) fp32 on the GPU -> uint16 tensor (H,W): nearest resize to `size` then *scale."""
    d = depth.reshape(depth.shape[-2:]).float().contiguous()
    H, W = d.shape
    OH, OW = (H, W) if size is None else size
    out = torch.empty((OH, OW), dtype=torch.uint16, device=d.device)
    ops.call('pf_depth_to_u16', d, H, W, OH, OW, C.c_float(scale), out, ops.stream_ptr())
    return out


def colormap_lut(cmap='gray_r'):
    """256 x 3 uint8 RGB lookup table.  'gray' / 'gray_r' are built with matplotlib's own recipe
    (`LinearSegmentedColormap` LUT = linspace(0,1,256), bytes = (lut*255).astype(uint8)); any other name (the
    reference's default 'magma_r', tester.py:69) is taken from matplotlib when it is installed."""
    if cmap in ('gray', 'gray_r'):
        ramp = np.linspace(0.0, 1.0, 256)
        if cmap.endswith('_r'):
            ramp = ramp[::-1]
        b = (ramp * 255).astype(np.uint8)
        return np.stack([b, b, b], 1).copy()
    try:
        import matplotlib
        cm = matplotlib.colormaps[cmap] if hasattr(matplotlib, 'colormaps') else matplotlib.cm.get_cmap(cmap)
    except Exception as e:           # pragma: no cover
        raise RuntimeError("colormap %r needs matplotlib (not installed here); use cmap='gray_r' "
                           "(the reference's --gray-scale path, tester.py:66-67)" % cmap) from e
    return (np.asarray(cm(np.linspace(0.0, 1.0, 256)))[:, :3] * 255).astype(np.uint8)


_LUTS = {}


def colorize(depth, cmap='magma_r', vmin=None, vmax=None, invalid_val=-99, vminp=2, vmaxp=95, bgr=False):
    """`estimator/utils/color.py:95-140` on the GPU: percentile normalisation (np.percentile semantics, linear
    interpolation, over the valid pixels; one device sort) + LUT lookup (pf_colorize_u8).  Returns uint8 (H, W, 3) on
    the device (RGB; BGR when bgr=True, i.e. the `[:, :, [2, 1, 0]]` the tester applies before cv2.imwrite)."""
    d = depth.reshape(depth.shape[-2:]).float().contiguous()
    key = (cmap, str(d.device))
    if key not in _LUTS:
        _LUTS[key] = torch.from_numpy(colormap_lut(cmap)).to(d.device).contiguous()
    if vmin is None or vmax is None:
        v = d.flatten()
        v = v[v != invalid_val]
        s, _ = torch.sort(v)
        n = s.numel()

        def pct(q):
            pos = (n - 1) * q / 100.0
            lo = int(np.floor(pos))
            hi = min(lo + 1, n - 1)
            a, b = s[lo].item(), s[hi].item()
            return a + (b - a) * (pos - lo)

        vmin = pct(vminp) if vmin is None else vmin
        vmax = pct(vmaxp) if vmax is None else vmax
    out = torch.empty(d.shape + (3,), dtype=torch.uint8, device=d.device)
    ops.call('pf_colorize_u8', d, C.c_int64(d.numel()), C.c_float(vmin), C.c_float(vmax), C.c_float(invalid_val),
             _LUTS[key], 1 if bgr else 0, out, ops.stream_ptr())
    return out
