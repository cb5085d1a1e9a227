"""CPU oracle for `BaselinePretrain.forward(mode='infer')` — TEST INFRASTRUCTURE, NOT PRODUCT.

A plain torch fp32 restatement of BP:333-419 (BP = estimator/models/baseline_pretrain.py of zhyever/PatchFusion) on
top of the helpers of oracle/pf_oracle.py (branch forward, tile plan, Gaussian mask, the literal RunningAverage):

    coarse target   branch_forward(sd, 'coarse_branch.', image_lr) at image_lr's own size
    fine target     regular passes of fine-branch tiles (no guided fusion) + N random_tile calls of process_num tiles

`build_baseline` instantiates the real reference `BaselinePretrain` from a shipped *_pretrain_u4k.py config through
oracle/shims; oracle/make_golden_baseline.py pins this restatement against it and writes tests/golden/vits_baseline0.*.
"""
import os
import random
import runpy

import numpy as np
import torch
import torch.nn.functional as F

from oracle import pf_oracle as po
from oracle import ref_harness as rh


def resize_da(x, size, multiple=14):
    """ResizeDA(w, h, keep_aspect_ratio=False, ensure_multiple_of=14, resize_method='minimal') (BP:75,85;
    depth_anything/transform.py:56-57,111-129): each side rounded to the nearest multiple, then bilinear
    align_corners=True."""
    H, W = x.shape[-2:]
    h = int(np.round(size[0] / H * H / multiple) * multiple)
    w = int(np.round(size[1] / W * W / multiple) * multiple)
    return po.up(x, (h, w))


class BaselineOracle:
    """BP:333-419 (mode='infer').  sd holds the prefixed keys of the built branch; cfg is the model dict of a
    *_pretrain_u4k.py config (patch_process_shape / image_raw_shape / patch_split_num default as in BP:51-53)."""

    def __init__(self, sd, cfg, target):
        assert target in ('coarse', 'fine')
        self.sd, self.cfg, self.target = sd, cfg, target
        self.P = tuple(po._get(cfg, 'patch_process_shape', (384, 512)))
        self.hp = po._get(cfg, target + '_branch')

    def resizer(self, x):
        return resize_da(x, self.P)

    def coarse(self, image_lr):
        """BP:366: one forward of the whole batch at its own size."""
        return po.branch_forward(self.sd, 'coarse_branch.', image_lr, self.hp)[0]

    def tiles(self, image_hr, raw_boxes, process_num, tile_cfg):
        """fine-branch depth (T,1,ph,pw) of the tiles with raw origins raw_boxes, in micro-batches (BP:293-308)."""
        h, w = tile_cfg['patch_raw_shape']
        crops = torch.cat([self.resizer(image_hr[:, :, y:y + h, x:x + w]) for (y, x) in raw_boxes])
        return torch.cat([po.branch_forward(self.sd, 'fine_branch.', crops[s:s + process_num], self.hp)[0]
                          for s in range(0, len(raw_boxes), process_num)])

    def infer(self, image_lr, image_hr, tile_cfg=None, cai_mode='m1', process_num=4):
        if self.target == 'coarse':
            return self.coarse(image_lr)
        cfg = self.cfg
        if tile_cfg is None:
            tile_cfg = dict(image_raw_shape=po._get(cfg, 'image_raw_shape', (2160, 3840)),
                            patch_split_num=po._get(cfg, 'patch_split_num', (4, 4)))
        tc = po.prepare_tile_cfg(tile_cfg['image_raw_shape'], tile_cfg['patch_split_num'], self.P)
        assert image_hr.shape[0] == 1
        dev = image_hr.device
        mask = torch.tensor(po.gaussian_mask(self.P) + 1e-3, device=dev)
        ph, pw = self.P
        RS = tc['patch_reensemble_shape']
        avg = None
        for pi, tiles in enumerate(po.tile_plan(tc, self.P, cai_mode)):
            preds = self.tiles(image_hr, [t[0] for t in tiles], process_num, tc)
            if pi == 0:                                       # init_flag=True (BP:315-317, 328-329)
                cnt, acc = torch.zeros(RS, device=dev), torch.zeros(RS, device=dev)
            for (_, (py, px)), d in zip(tiles, preds):
                if pi > 0:                                    # BP:319-324
                    cnt, acc = torch.zeros(RS, device=dev), torch.zeros(RS, device=dev)
                cnt[py:py + ph, px:px + pw] = mask
                acc[py:py + ph, px:px + pw] = d[0] * mask
                if pi > 0:
                    avg.update(acc, cnt)
            if pi == 0:
                avg = po.RunningAverage(acc, cnt)
        if cai_mode[0] == 'r':
            h, w = tc['patch_raw_shape']
            H, W = tc['image_raw_shape']
            mask = torch.tensor(po.gaussian_mask((h, w)) + 1e-3, device=dev)
            avg.resize((H, W))
            for _ in range(int(cai_mode[1:])):                # BP:407-410: N calls, not N // process_num
                ys = [random.randint(0, H - h - 1) for _ in range(process_num)]     # BP:155-156 draw order
                x0 = random.randint(0, W - w - 1)
                preds = F.interpolate(self.tiles(image_hr, [(y, x0) for y in ys], process_num, tc), (h, w))
                for y, d in zip(ys, preds):                   # BP:205-216
                    cnt, acc = torch.zeros((H, W), device=dev), torch.zeros((H, W), device=dev)
                    cnt[y:y + h, x0:x0 + w] = mask
                    acc[y:y + h, x0:x0 + w] = d[0] * mask
                    avg.update(acc, cnt)
        return avg.avg[None, None]


def baseline_config(encoder, target):
    """The model dict of configs/patchfusion_depthanything/depthanything_<enc>_<target>_pretrain_u4k.py with
    pretrained_resource=None on both branches (the configs point at local::./work_dir/... checkpoints)."""
    path = os.path.join(rh.REF, 'configs/patchfusion_depthanything/depthanything_%s_%s_pretrain_u4k.py'
                        % (encoder, target))
    model = dict(runpy.run_path(path)['model'])
    for b in ('coarse_branch', 'fine_branch'):
        model[b] = dict(model[b], pretrained_resource=None)
    return model


def build_baseline(encoder='vits', target='coarse', overrides=None):
    """Instantiate the reference BaselinePretrain (CPU, eval) from the shipped config's model dict + overrides."""
    rh._enter()
    from mmengine.config import ConfigDict
    cwd = os.getcwd()
    os.chdir(rh.REF)  # DPT:140 uses a relative torch.hub path
    try:
        import warnings
        warnings.filterwarnings('ignore')
        from estimator.models.baseline_pretrain import BaselinePretrain
        cfg = ConfigDict(baseline_config(encoder, target))
        cfg.update(overrides or {})
        cfg.pop('type')
        model = BaselinePretrain(**cfg).eval()
    finally:
        os.chdir(cwd)
    return model
