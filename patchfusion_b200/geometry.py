"""Depth to 3D on the GPU: the reference's geometry helpers (`external/zoedepth/utils/geometry.py`: get_intrinsics,
depth_to_points, create_triangles) on CUDA tensors, a vertex mask that drops the stretched triangles at depth
discontinuities, and a binary PLY writer.

Device tensors in, device tensors out; every pass is a kernel of csrc/pf_geom.cu, and torch only allocates.  A 4K
canvas gives 8.3 M vertices and up to 16.6 M triangles.

    from patchfusion_b200 import geometry
    verts, colors, faces = geometry.depth_to_mesh(depth[0], image_hr, edge_threshold=0.05)
    geometry.write_ply('mesh.ply', verts, colors, faces)

Batched depth [B, 1, H, W] is processed image by image; lists of depths of different sizes are handled by
depth_to_mesh one element at a time.
"""
import numpy as np
import torch

from . import ops

FOV_DEG = 55.0              # get_intrinsics' fixed field of view
MAX_VERTICES = 2 ** 31      # vertex indices are int32


def get_intrinsics(H, W):
    """K of geometry.py:27-37 (fp64 numpy): f = W / 2 / tan(27.5 deg), principal point (W/2, H/2)"""
    f = 0.5 * W / np.tan(0.5 * FOV_DEG * np.pi / 180.0)
    return np.array([[f, 0, 0.5 * W], [0, f, 0.5 * H], [0, 0, 1]])


def _check(t, name, dtypes, dims):
    """a contiguous CUDA tensor of one of `dtypes` with one of the ranks `dims`; raises before any launch"""
    if not isinstance(t, torch.Tensor):
        raise TypeError('%s must be a torch tensor, got %s' % (name, type(t).__name__))
    if not t.is_cuda:
        raise ValueError('%s must be on a CUDA device, got %s' % (name, t.device))
    if t.dtype not in dtypes:
        raise TypeError('%s must be %s, got %s' % (name, ' or '.join(str(d) for d in dtypes), t.dtype))
    if t.dim() not in dims:
        raise ValueError('%s must have %s dimensions, got shape %s' % (name, ' or '.join(map(str, dims)),
                                                                      tuple(t.shape)))
    if not t.is_contiguous():
        raise ValueError('%s must be contiguous' % name)


def _rt(R, t):
    """R [3, 3] and t [3] (array-likes, None: identity / zero) -> 12 host floats, or None for the identity"""
    if R is None and t is None:
        return None
    R = np.eye(3) if R is None else np.asarray(R.tolist() if isinstance(R, torch.Tensor) else R, dtype=np.float64)
    t = np.zeros(3) if t is None else np.asarray(t.tolist() if isinstance(t, torch.Tensor) else t, dtype=np.float64)
    if R.shape != (3, 3) or t.reshape(-1).shape != (3,):
        raise ValueError('R must be 3 x 3 and t of 3 elements, got %s and %s' % (R.shape, t.shape))
    return [float(v) for v in np.concatenate([R.reshape(-1), t.reshape(-1)]).astype(np.float32)]


def _inv_f(W):
    return float(np.float32(1.0 / get_intrinsics(1, W)[0, 0]))


def _images(depth, name='depth'):
    """depth [1, H, W] -> [depth]; [B, 1, H, W] -> its B images [1, H, W]"""
    _check(depth, name, (torch.float32,), (3, 4))
    if depth.shape[-3] != 1:
        raise ValueError('%s must be [1, H, W] or [B, 1, H, W], got %s' % (name, tuple(depth.shape)))
    return [depth] if depth.dim() == 3 else list(depth)


def depth_to_points(depth, R=None, t=None):
    """geometry.py:39-72 on the GPU: depth [1, H, W] fp32 -> points [H, W, 3] fp32, R M d K^-1 [x, y, 1]^T + t per
    pixel (M flips x and y).  depth [B, 1, H, W] -> [B, H, W, 3], image by image."""
    rt = _rt(R, t)
    imgs = _images(depth)
    H, W = depth.shape[-2:]
    out = torch.empty(depth.shape[:-3] + (H, W, 3), dtype=torch.float32, device=depth.device)
    with torch.cuda.device(depth.device):
        for d, o in zip(imgs, out.view(-1, H, W, 3)):
            ops.depth_to_points(d, _inv_f(W), rt, None, o)
    return out


def depth_edges_mask(depth, threshold):
    """Vertex mask [H, W] bool: hypot(d/dy, d/dx) <= threshold (threshold rounded to fp32), with the gradient of
    np.gradient in fp32 (central differences inside, one-sided at the borders); non-finite or non-positive depth is
    never kept.  depth [1, H, W] fp32, or [B, 1, H, W] -> [B, H, W]."""
    imgs = _images(depth)
    H, W = depth.shape[-2:]
    if H < 2 or W < 2:
        raise ValueError('depth_edges_mask needs at least 2 x 2 pixels (np.gradient), got %d x %d' % (H, W))
    out = torch.empty(depth.shape[:-3] + (H, W), dtype=torch.bool, device=depth.device)
    with torch.cuda.device(depth.device):
        for d, o in zip(imgs, out.view(-1, H, W)):
            ops.depth_edge_mask(d, float(threshold), o)
    return out


def create_triangles(h, w, mask=None, device=None):
    """geometry.py:75-98 on the GPU: triangle indices [n, 3] int32 of the h x w vertex grid, per quad (tl, bl, tr) then
    (br, tr, bl), quads row-major.  mask ([h, w] or [h * w], bool or uint8, on the device): keep a triangle only if
    its three vertices are set, in numpy's boolean-indexing order.  Without a mask the result is on `device` (default:
    the current CUDA device).  The masked path reads the triangle count back once to size the output."""
    h, w = int(h), int(w)
    if h < 2 or w < 2:
        raise ValueError('create_triangles needs at least 2 x 2 vertices, got %d x %d' % (h, w))
    if h * w >= MAX_VERTICES:
        raise ValueError('create_triangles: %d x %d vertices do not fit int32 indices' % (h, w))
    if mask is not None:
        if not isinstance(mask, torch.Tensor) or tuple(mask.shape) not in ((h, w), (h * w,)):
            raise ValueError('mask must be a tensor of shape (%d, %d), got %s' %
                             (h, w, tuple(mask.shape) if isinstance(mask, torch.Tensor) else type(mask).__name__))
        _check(mask, 'mask', (torch.bool, torch.uint8), (1, 2))
        device = mask.device
    device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    nq = (h - 1) * (w - 1)
    with torch.cuda.device(device):
        if mask is None:
            faces = torch.empty((2 * nq, 3), dtype=torch.int32, device=device)
            ops.mesh_triangles(None, None, h, w, faces)
            return faces
        nb = ops.mesh_scan_blocks(h, w)
        flags = torch.empty(nq, dtype=torch.uint8, device=device)
        offsets = torch.empty(nb + 1, dtype=torch.int64, device=device)
        ops.mesh_quad_counts(mask, h, w, flags, offsets)
        n = int(offsets[nb].item())
        faces = torch.empty((n, 3), dtype=torch.int32, device=device)
        if n:
            ops.mesh_triangles(flags, offsets, h, w, faces)
    return faces


def depth_to_mesh(depth, image=None, edge_threshold=None, R=None, t=None):
    """depth [1, H, W] fp32 -> (vertices [H*W, 3] fp32, colors [H*W, 3] uint8 or None, faces [n, 3] int32), all on the
    device.  image: the [1, 3, H, W] fp32 image_hr in [0, 1]; colours are round(255 clamp(v, 0, 1)), written by the
    pass that writes the points.  edge_threshold: drop triangles touching a vertex depth_edges_mask rejects.
    depth [B, 1, H, W] (with image [B, 3, H, W]) or a list of depths (with a list of images) -> list of meshes."""
    if isinstance(depth, (list, tuple)) or depth.dim() == 4:
        images = [None] * len(depth) if image is None else list(image)
        if len(images) != len(depth):
            raise ValueError('%d depths but %d images' % (len(depth), len(images)))
        return [depth_to_mesh(d, im, edge_threshold, R, t) for d, im in zip(depth, images)]
    rt = _rt(R, t)
    (depth,) = _images(depth)
    H, W = depth.shape[-2:]
    if image is not None:
        _check(image, 'image', (torch.float32,), (3, 4))
        if tuple(image.shape[-3:]) != (3, H, W) or image.numel() != 3 * H * W:
            raise ValueError('image must be [1, 3, %d, %d], got %s' % (H, W, tuple(image.shape)))
        if image.device != depth.device:
            raise ValueError('image is on %s, depth on %s' % (image.device, depth.device))
    points = torch.empty((H * W, 3), dtype=torch.float32, device=depth.device)
    colors = None if image is None else torch.empty((H * W, 3), dtype=torch.uint8, device=depth.device)
    with torch.cuda.device(depth.device):
        ops.depth_to_points(depth, _inv_f(W), rt, image, points, colors)
    mask = None if edge_threshold is None else depth_edges_mask(depth, edge_threshold)
    faces = create_triangles(H, W, mask, device=depth.device)
    return points, colors, faces


def _ply_header(nv, nf, color):
    lines = ['ply', 'format binary_little_endian 1.0', 'element vertex %d' % nv,
             'property float x', 'property float y', 'property float z']
    if color:
        lines += ['property uchar red', 'property uchar green', 'property uchar blue']
    lines += ['element face %d' % nf, 'property list uchar int vertex_indices', 'end_header']
    return ('\n'.join(lines) + '\n').encode('ascii')


PLY_VERTEX = np.dtype([('xyz', '<f4', (3,))])
PLY_VERTEX_RGB = np.dtype([('xyz', '<f4', (3,)), ('rgb', 'u1', (3,))])      # 15 bytes, unpadded
PLY_FACE = np.dtype([('n', 'u1'), ('v', '<i4', (3,))])                      # 13 bytes, unpadded


def _to_host(t):
    """one pinned D2H copy of a contiguous device tensor, as a numpy byte array (after the stream synchronises)"""
    host = torch.empty(t.numel() * t.element_size(), dtype=torch.uint8, pin_memory=True)
    if host.numel():
        host.copy_(t.reshape(-1).view(torch.uint8), non_blocking=True)
    return host


def _pack_device(vertices, colors, faces):
    dev = vertices.device
    with torch.cuda.device(dev):
        if colors is None:
            vbytes = vertices
        else:
            vbytes = torch.empty(15 * vertices.shape[0], dtype=torch.uint8, device=dev)
            if vertices.shape[0]:
                ops.ply_pack_vertices(vertices, colors, vbytes)
        fbytes = torch.empty(13 * faces.shape[0], dtype=torch.uint8, device=dev)
        if faces.shape[0]:
            ops.ply_pack_faces(faces, fbytes)
        hv, hf = _to_host(vbytes), _to_host(fbytes)
        torch.cuda.current_stream().synchronize()
    return hv.numpy(), hf.numpy()


def _pack_host(vertices, colors, faces):
    v = np.asarray(vertices, dtype=np.float32).reshape(-1, 3)
    rec = np.empty(v.shape[0], PLY_VERTEX if colors is None else PLY_VERTEX_RGB)
    rec['xyz'] = v
    if colors is not None:
        rec['rgb'] = np.asarray(colors, dtype=np.uint8).reshape(-1, 3)
    f = np.asarray(faces).reshape(-1, 3)
    if f.size and (f.min() < 0 or f.max() >= MAX_VERTICES):
        raise ValueError('face indices must be in [0, 2^31)')
    frec = np.empty(f.shape[0], PLY_FACE)
    frec['n'] = 3
    frec['v'] = f
    return rec.view(np.uint8), frec.view(np.uint8)


def write_ply(path, vertices, colors, faces):
    """Binary little-endian PLY: float x, y, z, optional uchar red, green, blue, and faces as a uchar count (3) plus
    int32 indices.  vertices [N, 3] (or [H, W, 3]) fp32, colors [N, 3] uint8 or None, faces [n, 3] int32 or None.
    Device tensors are packed into PLY records on the GPU and each array comes back in one pinned copy; host arrays
    (numpy or CPU tensors) are laid out with numpy."""
    faces = torch.empty((0, 3), dtype=torch.int32, device=vertices.device if isinstance(vertices, torch.Tensor)
                        else 'cpu') if faces is None else faces
    on_device = [isinstance(a, torch.Tensor) and a.is_cuda for a in (vertices, colors, faces) if a is not None]
    if any(on_device):
        if not all(on_device):
            raise ValueError('write_ply: vertices, colors and faces must all be on the device or all on the host')
        _check(vertices, 'vertices', (torch.float32,), (2, 3))
        vertices = vertices.view(-1, 3)
        if colors is not None:
            _check(colors, 'colors', (torch.uint8,), (2, 3))
            colors = colors.view(-1, 3)
        _check(faces, 'faces', (torch.int32,), (2,))
        if (colors is not None and colors.shape != vertices.shape) or faces.shape[-1] != 3:
            raise ValueError('write_ply: colors must match vertices [N, 3] and faces be [n, 3]')
        if len({vertices.device, faces.device} | ({colors.device} if colors is not None else set())) != 1:
            raise ValueError('write_ply: the arrays are on different devices')
        vb, fb = _pack_device(vertices, colors, faces)
    else:
        vb, fb = _pack_host(*(a.numpy() if isinstance(a, torch.Tensor) else a for a in (vertices, colors, faces)))
    nv = vb.size // (12 if colors is None else 15)
    with open(path, 'wb') as f:
        f.write(_ply_header(nv, fb.size // 13, colors is not None))
        f.write(memoryview(vb))
        f.write(memoryview(fb))
    return path
