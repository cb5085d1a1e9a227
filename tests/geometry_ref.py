"""Host references for patchfusion_b200/geometry.py: `external/zoedepth/utils/geometry.py` restated in numpy fp64
(pinned to the reference by tests/golden/geometry_case0.npz), the np.gradient vertex mask, the colour rounding and a
small binary PLY reader."""
import numpy as np


def get_intrinsics(H, W):
    f = 0.5 * W / np.tan(0.5 * 55 * np.pi / 180.0)
    return np.array([[f, 0, 0.5 * W], [0, f, 0.5 * H], [0, 0, 1]], dtype=np.float64)


def depth_to_points(depth, R=None, t=None):
    """depth [1, H, W] -> points [H, W, 3] fp64: R M d K^-1 [x, y, 1]^T + t, M = diag(-1, -1, 1)"""
    d = np.asarray(depth, dtype=np.float64)
    _, H, W = d.shape
    R = np.eye(3) if R is None else np.asarray(R, dtype=np.float64)
    t = np.zeros(3) if t is None else np.asarray(t, dtype=np.float64).reshape(3)
    y, x = np.mgrid[0:H, 0:W]
    coord = np.stack([x, y, np.ones_like(x)], -1).astype(np.float64)
    p = d[0][..., None] * (coord @ np.linalg.inv(get_intrinsics(H, W)).T)
    p = p * np.array([-1.0, -1.0, 1.0])
    return p @ R.T + t


def create_triangles(h, w, mask=None):
    """int64 [n, 3]: per quad (tl, bl, tr), (br, tr, bl), quads row-major; with a mask, the triangles whose three
    vertices are set, in boolean-indexing order"""
    y, x = np.mgrid[0:h - 1, 0:w - 1].astype(np.int64)
    tl = y * w + x
    tri = np.stack([tl, tl + w, tl + 1, tl + w + 1, tl + 1, tl + w], -1).reshape(-1, 3)
    if mask is not None:
        tri = tri[np.asarray(mask).reshape(-1).astype(bool)[tri].all(1)]
    return tri


def edge_mask(depth, threshold):
    """[H, W] bool: finite d > 0 and hypot(np.gradient(d)) <= fp32(threshold), all in fp32"""
    d = np.asarray(depth, dtype=np.float32)
    d = d.reshape(d.shape[-2:])
    with np.errstate(invalid='ignore', over='ignore'):
        gy, gx = np.gradient(d)
        g = np.hypot(gy, gx)
        return np.isfinite(d) & (d > 0) & (g <= np.float32(threshold))


def gradient_norm(depth):
    d = np.asarray(depth, dtype=np.float32)
    with np.errstate(invalid='ignore', over='ignore'):
        gy, gx = np.gradient(d.reshape(d.shape[-2:]))
        return np.hypot(gy, gx)


def colors(image):
    """planar [.., 3, H, W] fp32 -> [H*W, 3] uint8 round-half-even(255 clamp(v, 0, 1)) in fp32"""
    v = np.asarray(image, dtype=np.float32).reshape(3, -1).T
    return np.rint(np.float32(255) * np.clip(v, np.float32(0), np.float32(1))).astype(np.uint8)


def read_ply(path):
    """binary little-endian PLY with float x, y, z, optional uchar red, green, blue and uchar-counted int32 faces ->
    dict(vertices [N, 3] fp32, colors [N, 3] uint8 or None, faces [n, 3] int32, counts (N, n), header lines)"""
    data = open(path, 'rb').read()
    end = data.index(b'end_header\n') + len(b'end_header\n')
    header = data[:end].decode('ascii').splitlines()
    assert header[0] == 'ply' and header[1] == 'format binary_little_endian 1.0', header[:2]
    counts, props, element = {}, {'vertex': [], 'face': []}, None
    for line in header[2:-1]:
        tok = line.split()
        if tok[0] == 'element':
            element = tok[1]
            counts[element] = int(tok[2])
        elif tok[0] == 'property':
            props[element].append(tuple(tok[1:]))
    xyz = [('float', 'x'), ('float', 'y'), ('float', 'z')]
    rgb = [('uchar', 'red'), ('uchar', 'green'), ('uchar', 'blue')]
    assert props['vertex'] in (xyz, xyz + rgb), props['vertex']
    assert props['face'] == [('list', 'uchar', 'int', 'vertex_indices')], props['face']
    has_rgb = props['vertex'] == xyz + rgb
    vt = np.dtype([('xyz', '<f4', (3,))] + ([('rgb', 'u1', (3,))] if has_rgb else []))
    ft = np.dtype([('n', 'u1'), ('v', '<i4', (3,))])
    nv, nf = counts['vertex'], counts['face']
    assert len(data) == end + nv * vt.itemsize + nf * ft.itemsize, 'file size does not match the header counts'
    v = np.frombuffer(data, vt, nv, end)
    f = np.frombuffer(data, ft, nf, end + nv * vt.itemsize)
    assert (f['n'] == 3).all()
    return dict(vertices=v['xyz'].copy(), colors=v['rgb'].copy() if has_rgb else None, faces=f['v'].copy(),
                counts=(nv, nf), header=header)
