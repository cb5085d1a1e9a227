"""Seeded synthetic evaluation data in the reference's on-disk layouts, for tests, fixtures and the evaluation
benchmark: a U4K split (raw frames, .npy disparities, Extrinsics0/1 files), a Middlebury pair (PFM + calib), an ETH3D
raw depth and a Cityscapes uint16 disparity PNG.  Every map holds the values that stress the ground-truth transforms:
zeros, +-inf, NaN and neighbour steps of exactly +-1 (the edge threshold)."""
import os
import os.path as osp

import numpy as np

from .datasets import ETH3D_SHAPE, U4K_SHAPE


def _stress(d, rng, lo, hi):
    """piecewise-constant float32 map with exact +-1 steps, zeros, infs and NaNs at seeded places"""
    H, W = d.shape
    d[:] = rng.uniform(lo, hi, size=(H, W)).astype(np.float32)
    by, bx = max(H // 16, 1), max(W // 16, 1)
    for _ in range(24):                                       # constant blocks: steps only at block borders
        y, x = int(rng.integers(0, H)), int(rng.integers(0, W))
        d[y:y + by, x:x + bx] = np.float32(rng.uniform(lo, hi))
    for _ in range(8):                                        # exact +-1 steps (|delta| == th: no edge)
        y, x = int(rng.integers(0, H)), int(rng.integers(0, max(W - bx, 1)))
        v = np.float32(np.round(rng.uniform(lo + 1, hi - 1)))
        d[y:y + by, x:x + bx // 2] = v
        d[y:y + by, x + bx // 2:x + bx] = v + np.float32(1) if rng.integers(0, 2) else v - np.float32(1)
    for val in (0.0, np.inf, -np.inf, np.nan):
        for _ in range(3):
            y, x = int(rng.integers(0, H)), int(rng.integers(0, W))
            d[y:y + 3, x:x + 5] = val
    d[0, 0], d[-1, -1] = 0.0, np.inf                          # image corners
    return d


def u4k_disparity(seed, shape=U4K_SHAPE):
    return _stress(np.empty(shape, np.float32), np.random.default_rng(seed), 0.5, 60.0)


def u4k_frame(seed, shape=U4K_SHAPE):
    return np.random.default_rng(seed + 1000).integers(0, 256, size=shape + (3,), dtype=np.uint8)


def write_u4k_tree(root, n, seed=0, scenes=('00001', '00000')):
    """root/<scene>/{Image0,Image1,Disp0,Disp1,Extrinsics0,Extrinsics1}/<k>.* and root/splits/val.txt listing n left
    images spread over the scenes, in an order that is not sorted.  Returns the split path."""
    lines = []
    for i in range(n):
        scene, k = scenes[i % len(scenes)], '%05d' % (n - i)
        for sub in ('Image0', 'Image1', 'Disp0', 'Disp1', 'Extrinsics0', 'Extrinsics1'):
            os.makedirs(osp.join(root, scene, sub), exist_ok=True)
        u4k_frame(seed + i).tofile(osp.join(root, scene, 'Image0', k + '.raw'))
        np.save(osp.join(root, scene, 'Disp0', k + '.npy'), u4k_disparity(seed + i))
        rng = np.random.default_rng(seed + 2000 + i)
        f, tx0 = rng.uniform(1500, 2500), rng.uniform(-1, 1)
        tx1 = tx0 + rng.uniform(0.2, 0.8)
        for sub, tx in (('Extrinsics0', tx0), ('Extrinsics1', tx1)):
            with open(osp.join(root, scene, sub, k + '.txt'), 'w') as fe:
                fe.write('%r 0 1920 0\n1 0 0 %r\n0 1 0 0\n0 0 1 0\n' % (f, tx))
        lines.append('%s/Image0/%s.png %s/Image1/%s.png %s/Disp0/%s.npy %s/Disp1/%s.npy' %
                     ((scene, k) * 4))
    os.makedirs(osp.join(root, 'splits'), exist_ok=True)
    split = osp.join(root, 'splits', 'val.txt')
    with open(split, 'w') as f:
        f.write('\n'.join(lines) + '\n')
    return split


def mid_disparity(seed, shape=(300, 437)):
    return _stress(np.empty(shape, np.float32), np.random.default_rng(seed), 20.0, 250.0)


def write_pfm(path, data):
    """little-endian greyscale PFM, rows stored bottom-up"""
    H, W = data.shape
    with open(path, 'wb') as f:
        f.write(b'Pf\n%d %d\n-1.0\n' % (W, H))
        np.flipud(data).astype('<f4').tofile(f)


def write_mid_tree(root, seed=0):
    """root/{images,gts,calibs}/mid0.{png,pfm,txt}"""
    import cv2
    for sub in ('images', 'gts', 'calibs'):
        os.makedirs(osp.join(root, sub), exist_ok=True)
    d = mid_disparity(seed)
    cv2.imwrite(osp.join(root, 'images', 'mid0.png'), u4k_frame(seed, d.shape))
    write_pfm(osp.join(root, 'gts', 'mid0.pfm'), d)
    with open(osp.join(root, 'calibs', 'mid0.txt'), 'w') as f:
        f.write('cam0=[3997.684 0 1176.728; 0 3997.684 1011.728; 0 0 1]\n'
                'cam1=[3997.684 0 1307.839; 0 3997.684 1011.728; 0 0 1]\ndoffs=131.111\nbaseline=193.001\n'
                'width=2964\nheight=1988\nndisp=280\n')


def eth3d_depth(seed, shape=ETH3D_SHAPE):
    return _stress(np.empty(shape, np.float32), np.random.default_rng(seed), 0.5, 30.0)


def write_eth3d_tree(root, seed=0):
    """root/{images,gts}/eth0.{png,raw}"""
    import cv2
    for sub in ('images', 'gts'):
        os.makedirs(osp.join(root, sub), exist_ok=True)
    cv2.imwrite(osp.join(root, 'images', 'eth0.png'), u4k_frame(seed, (64, 96)))
    eth3d_depth(seed).tofile(osp.join(root, 'gts', 'eth0.raw'))


def cityscapes_disparity(seed, shape=(256, 512)):
    rng = np.random.default_rng(seed)
    d = rng.integers(0, 30000, size=shape).astype(np.uint16)
    d[rng.random(shape) < 0.05] = 0
    d[rng.random(shape) < 0.05] = 1                 # (1 - 1) / 256 = 0 -> inf -> 0
    d[10:20, 10:40] = 5000
    d[10:20, 40:70] = 5256                          # a step of exactly 1 in (x - 1) / 256
    return d


def write_cityscapes_tree(root, seed=0):
    """root/{images,gts}/city0.png (uint16 disparity)"""
    import cv2
    for sub in ('images', 'gts'):
        os.makedirs(osp.join(root, sub), exist_ok=True)
    d = cityscapes_disparity(seed)
    cv2.imwrite(osp.join(root, 'images', 'city0.png'), u4k_frame(seed, d.shape))
    cv2.imwrite(osp.join(root, 'gts', 'city0.png'), d)


def write_u4k_case(root, n_frames, encoder='vits', split_num=(2, 2), seed=3):
    """A U4K tree of n_frames, seeded synthetic weights saved as a .pth checkpoint and a reference-format config whose
    val_dataloader reads the tree.  Returns (config path, checkpoint path, model config dict)."""
    import torch
    from .configs import depth_anything_patchfusion
    from .params import synthetic_state_dict
    split = write_u4k_tree(osp.join(root, 'u4k'), n_frames, seed=seed)
    cfg = depth_anything_patchfusion(encoder, image_raw_shape=U4K_SHAPE, patch_split_num=split_num)
    ckpt = osp.join(root, 'ckpt', '%s_synthetic.pth' % encoder)
    os.makedirs(osp.dirname(ckpt), exist_ok=True)
    torch.save({'model_state_dict': synthetic_state_dict(cfg, seed=0)}, ckpt)
    conf = osp.join(root, 'cfg_%s_u4k.py' % encoder)
    with open(conf, 'w') as f:
        f.write('model = dict(type="PatchFusion", config=%r)\n'
                'val_dataloader = dict(batch_size=1, num_workers=2, dataset=dict(type="UnrealStereo4kDataset", '
                'mode="infer", data_root=%r, split=%r, min_depth=1e-3, max_depth=80, '
                'transform_cfg=dict(network_process_size=[392, 518]), resize_mode="depth-anything"))\n'
                % (cfg, osp.join(root, 'u4k'), split))
    return conf, ckpt, cfg
