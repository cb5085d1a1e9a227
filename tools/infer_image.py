"""Counterpart of the reference's tools/test_single_forward.py on the CUDA path: image file (or synthetic) -> GPU ingest
-> PatchFusion.forward -> uint16 depth PNG, and with --mesh a coloured PLY mesh of the depth (patchfusion_b200/geometry.py).
Weights: a HF/local checkpoint directory via --model, else seeded synthetic.

    python tools/infer_image.py --image examples/example_1.jpeg --out depth_u16.png --mode r128 --encoder vitl
    python tools/infer_image.py --image examples/example_1.jpeg --mesh out.ply --edge-threshold 0.05
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from patchfusion_b200 import geometry, imageio, ops
from patchfusion_b200.configs import depth_anything_patchfusion
from patchfusion_b200.model import PatchFusion

ap = argparse.ArgumentParser()
ap.add_argument('--image', default=None)
ap.add_argument('--model', default=None, help='directory or hub id for PatchFusion.from_pretrained')
ap.add_argument('--encoder', default='vitl')
ap.add_argument('--mode', default='m2')
ap.add_argument('--process-num', type=int, default=9)
ap.add_argument('--raw-shape', type=int, nargs=2, default=[2160, 3840])
ap.add_argument('--split', type=int, nargs=2, default=[4, 4])
ap.add_argument('--out', default='depth_u16.png')
ap.add_argument('--mesh', default=None, help='also write the mesh of the depth at --raw-shape to this .ply file')
ap.add_argument('--edge-threshold', type=float, default=None,
                help='drop mesh triangles at vertices whose depth-gradient norm exceeds this (metres per pixel)')
a = ap.parse_args()
dev = torch.device('cuda:0')
if a.model:
    model = PatchFusion.from_pretrained(a.model)
else:
    model = PatchFusion(depth_anything_patchfusion(a.encoder, tuple(a.raw_shape), tuple(a.split))).init_synthetic_weights(0)
model = model.to(dev).eval()
if a.image:
    import cv2
    bgr = cv2.imread(a.image)
    h0, w0 = bgr.shape[:2]
else:
    bgr = np.random.default_rng(0).integers(0, 256, (1080, 1920, 3), dtype=np.uint8)
    h0, w0 = 1080, 1920
image = imageio.ingest(bgr, tuple(a.raw_shape), dev, bgr=True)
image_lr = model.make_lr(image)
tile_cfg = {'image_raw_shape': list(a.raw_shape), 'patch_split_num': list(a.split)}
depth, _ = model(mode='infer', cai_mode=a.mode, process_num=a.process_num, image_lr=image_lr, image_hr=image, tile_cfg=tile_cfg)
u16 = imageio.depth_to_u16(depth, (h0, w0)).cpu().numpy()
try:
    import cv2
    cv2.imwrite(a.out, u16)
except Exception:
    np.save(a.out + '.npy', u16)
print('depth', tuple(depth.shape), 'range %.3f..%.3f' % (depth.min().item(), depth.max().item()), '->', a.out)
if a.mesh:
    # the canvas is at the tiles' network resolution: bring it to image_raw_shape (bilinear, align_corners=True), the
    # grid of the ingested image that colours the vertices
    mesh_depth = torch.empty((1,) + tuple(a.raw_shape), dtype=torch.float32, device=dev)
    ops.call('pf_resize_bilinear_f32', depth, 1, depth.shape[-2], depth.shape[-1], 1, a.raw_shape[0], a.raw_shape[1],
             mesh_depth, ops.stream_ptr())
    verts, colors, faces = geometry.depth_to_mesh(mesh_depth, image, edge_threshold=a.edge_threshold)
    geometry.write_ply(a.mesh, verts, colors, faces)
    print('mesh', '%d vertices (%d x %d)' % (verts.shape[0], a.raw_shape[0], a.raw_shape[1]),
          '%d faces' % faces.shape[0], '->', a.mesh)
