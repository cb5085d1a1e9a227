"""Runs the reference's own evaluation datasets (`estimator/datasets/u4k_dataset.py`, `general_dataset.py`, imported
unmodified through oracle/shims, build container only) on the seeded synthetic tree of patchfusion_b200/eval_tree.py
and writes tests/golden/eval_case0.{json,npz}: the U4K data_infos and basenames, strided samples plus full corner and
centre crops of depth_gt / boundary for u4k, mid, eth3d and cityscapes and of the U4K image_hr, and the reference's
compute_metrics (with a finite soft edge error) of a fixed prediction against each U4K depth_gt.  It also checks
load_config on the three depthanything_*_patchfusion_u4k.py configs against
patchfusion_b200.configs.depth_anything_patchfusion.

    PATCHFUSION_REFERENCE=<checkout> python -m oracle.make_golden_eval
"""
import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import ref_harness as rh                 # noqa: E402
from patchfusion_b200 import eval_tree as et          # noqa: E402

U4K_N = 3
CROP = 24


def sample_index(shape, target=12000):
    """flat indices: a stride over the whole map plus full CROP x CROP crops at the four corners and the centre"""
    H, W = shape
    idx = set(range(0, H * W, max(H * W // target, 1)))
    for y0 in (0, H - CROP, (H - CROP) // 2):
        for x0 in (0, W - CROP, (W - CROP) // 2):
            for y in range(max(y0, 0), min(y0 + CROP, H)):
                idx.update(range(y * W + max(x0, 0), y * W + min(x0 + CROP, W)))
    return np.array(sorted(idx), dtype=np.int64)


def _np(x):
    return x.numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


def fixed_prediction(shape, seed=7):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(1, 1, shape[0] // 4, shape[1] // 4, generator=g) * 70 + 0.5


def normalized(v):
    if isinstance(v, dict):
        return {k: normalized(x) for k, x in v.items()}
    if isinstance(v, (list, tuple)):
        return [normalized(x) for x in v]
    return v


def check_configs():
    from patchfusion_b200.config import load_config
    from patchfusion_b200.configs import depth_anything_patchfusion
    for enc in ('vits', 'vitb', 'vitl'):
        cfg = load_config(os.path.join(rh.REF, 'configs/patchfusion_depthanything/'
                                       'depthanything_%s_patchfusion_u4k.py' % enc))
        got, want = normalized(cfg.model.config.to_dict()), normalized(depth_anything_patchfusion(enc))
        for k in want:
            if k in ('load_branch', 'pretrain_model'):      # where the training run kept its branch checkpoints
                continue
            if k in ('coarse_branch', 'fine_branch'):
                assert {a: got[k][a] for a in want[k]} == want[k], (enc, k)
            else:
                assert got[k] == want[k], (enc, k, got[k], want[k])
        print('config', enc, 'ok')


def main():
    check_configs()
    rh._enter()
    import estimator.datasets.utils as ref_utils
    ref_utils.sys = sys                       # readPFM reads sys.version, which that module never imports
    from estimator.datasets.general_dataset import DepthMap
    from estimator.datasets.u4k_dataset import UnrealStereo4kDataset
    from estimator.utils.metric import compute_metrics
    from mmengine.config import ConfigDict

    js, arrays = {}, {}
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, 'u4k')
        split = et.write_u4k_tree(root, U4K_N, seed=0)
        ds = UnrealStereo4kDataset(mode='infer', data_root=root, split=split,
                                   transform_cfg=ConfigDict(network_process_size=[392, 518]), min_depth=1e-3,
                                   max_depth=80, resize_mode='depth-anything')
        js['u4k_split'] = open(split).read()
        js['u4k_infos'] = [dict(img_path=os.path.relpath(i['img_path'], root),
                                depth_map_path=os.path.relpath(i['depth_map_path'], root), filename=i['filename'],
                                focal=i['focal'], depth_factor=i['depth_factor']) for i in ds.data_infos]
        js['u4k_basenames'], js['u4k_metrics'] = [], []
        for i in range(U4K_N):
            s = ds[i]
            js['u4k_basenames'].append(s['img_file_basename'])
            depth, boundary, image = _np(s['depth_gt'])[0], _np(s['boundary'])[0], _np(s['image_hr'])
            idx = sample_index(depth.shape)
            arrays['u4k%d_idx' % i] = idx
            arrays['u4k%d_depth' % i] = depth.reshape(-1)[idx]
            arrays['u4k%d_boundary' % i] = boundary.reshape(-1)[idx]
            arrays['u4k%d_image' % i] = image.reshape(3, -1)[:, idx]
            pred = fixed_prediction(depth.shape)
            # NaN depth (NaN disparity) zeroed: a NaN neighbour turns the reference's soft edge error into NaN
            gt = torch.nan_to_num(s['depth_gt'], nan=0.0, posinf=float('inf'), neginf=float('-inf'))
            m = compute_metrics(gt[None], pred.clone(), disp_gt_edges=s['boundary'], min_depth_eval=1e-3,
                                max_depth_eval=80, garg_crop=False, eigen_crop=False, dataset='')
            assert np.isfinite(float(m['see'])), m
            js['u4k_metrics'].append({k: float(v) for k, v in m.items()})

        for name, writer, gt_name in (('mid', et.write_mid_tree, 'mid0.pfm'), ('eth3d', et.write_eth3d_tree, 'eth0.raw'),
                                      ('cityscapes', et.write_cityscapes_tree, 'city0.png')):
            sub = os.path.join(tmp, name)
            writer(sub, seed=0)
            dm = DepthMap(os.path.join(sub, 'gts'), [gt_name], 0, name)
            depth, boundary = np.asarray(dm.gt, np.float32), np.asarray(dm.edge, np.float32)
            idx = sample_index(depth.shape)
            arrays['%s_idx' % name] = idx
            arrays['%s_depth' % name] = depth.reshape(-1)[idx]
            arrays['%s_boundary' % name] = boundary.reshape(-1)[idx]
            js['%s_shape' % name] = list(depth.shape)
            js['%s_name' % name] = dm.name
    json.dump(js, open(os.path.join(ROOT, 'tests', 'golden', 'eval_case0.json'), 'w'), indent=1)
    np.savez_compressed(os.path.join(ROOT, 'tests', 'golden', 'eval_case0.npz'), **arrays)
    print('wrote eval_case0', {k: v.shape for k, v in arrays.items()})


if __name__ == '__main__':
    main()
