"""Pins oracle/baseline_oracle.py against the real reference BaselinePretrain and writes tests/golden/vits_baseline0.*.

Needs a zhyever/PatchFusion checkout:   PATCHFUSION_REFERENCE=<checkout> python -m oracle.make_golden_baseline

Case: the 1080x1920 image of vits_case0, patch_split_num (2, 2), process_num 2; the weights are the coarse_branch.* /
fine_branch.* subsets of synthetic_state_dict(depth_anything_patchfusion('vits'), 0), loaded through the reference's
own `load_dict`.  The coarse target is built from the shipped coarse config as it is (patch_process_shape keeps the
(384, 512) default) and run at B = 2 at two sizes: the reference's own resizer(img) (378x518) and the dataset size
392x518.  The fine target runs m1, m2 and r4 (random.seed(0) before each).
"""
import json
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from oracle import baseline_oracle as bo                             # noqa: E402
from oracle.make_golden import CASE, case_inputs, sample, save_parts  # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden')


def unprefixed(sd, prefix):
    return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}


def check_layout(ref_model, prefix):
    layout = json.load(open(os.path.join(GOLD, 'state_dict_layout_vits.json')))
    want = [(k, v[0], v[1]) for k, v in layout.items() if k.startswith(prefix)]
    got = [(k, list(v.shape), str(v.dtype).replace('torch.', '')) for k, v in ref_model.state_dict().items()]
    assert got == want, 'reference state_dict() differs from the %s* subset of the PatchFusion layout' % prefix


def report(tag, ref, got, tol):
    err = (ref - got).abs().max().item()
    print('%-28s %s max|ref-oracle| = %.3e (range %.3f..%.3f)' % (tag, tuple(ref.shape), err, ref.min().item(),
                                                                   ref.max().item()))
    assert err < tol * ref.abs().max().item(), tag


def main():
    torch.set_num_threads(os.cpu_count())
    case = dict(CASE, name='vits_baseline0', lr_sizes=[[378, 518], [392, 518]], coarse_batch=2)
    cfg, sd, img = case_inputs(case)
    split = dict(image_raw_shape=tuple(case['image_raw_shape']), patch_split_num=tuple(case['patch_split_num']))
    g = torch.Generator().manual_seed(case['input_seed'] + 1)
    img2 = torch.rand(1, 3, *case['image_raw_shape'], generator=g)      # second image of the coarse batch
    out, st = {}, case['sample_stride']
    with torch.no_grad():
        # ---- coarse target: the shipped config as it is (default patch_process_shape (384, 512))
        ref = bo.build_baseline(case['encoder'], 'coarse')
        check_layout(ref, 'coarse_branch.')
        print('coarse load_dict:', ref.load_dict(unprefixed(sd, 'coarse_branch.')))
        orc = bo.BaselineOracle(sd, bo.baseline_config(case['encoder'], 'coarse'), 'coarse')
        lr = ref.resizer(torch.cat([img, img2]))
        assert tuple(lr.shape[-2:]) == tuple(case['lr_sizes'][0]), lr.shape
        assert torch.equal(lr, orc.resizer(torch.cat([img, img2])))
        for size in case['lr_sizes']:
            x = lr if list(lr.shape[-2:]) == size else torch.nn.functional.interpolate(
                torch.cat([img, img2]), tuple(size), mode='bilinear', align_corners=True)
            y_ref, info = ref(mode='infer', image_lr=x, image_hr=None, depth_gt=None)
            assert set(info) == {'rgb', 'depth_pred', 'depth_gt'}
            report('coarse %dx%d' % tuple(size), y_ref, orc.infer(x, None), 1e-5)
            out['coarse_%dx%d' % tuple(size)] = sample(y_ref, st)
        del ref
        # ---- fine target
        ref = bo.build_baseline(case['encoder'], 'fine', split)
        check_layout(ref, 'fine_branch.')
        print('fine load_dict:', ref.load_dict(unprefixed(sd, 'fine_branch.')))
        save = ref.get_save_dict()
        assert list(save) == list(unprefixed(sd, 'fine_branch.'))
        fcfg = dict(bo.baseline_config(case['encoder'], 'fine'), **split)
        orc = bo.BaselineOracle(sd, fcfg, 'fine')
        for mode in ('m1', 'm2', 'r4'):
            random.seed(0)
            y_ref, info = ref(mode='infer', image_lr=None, image_hr=img, depth_gt=None, cai_mode=mode,
                              process_num=case['process_num'])
            assert info == {}
            random.seed(0)
            report('fine ' + mode, y_ref, orc.infer(None, img, cai_mode=mode, process_num=case['process_num']), 1e-3)
            out['fine_' + mode] = sample(y_ref, st)
    os.makedirs(GOLD, exist_ok=True)
    save_parts(os.path.join(GOLD, 'vits_baseline0'), out)
    json.dump({k: (list(v) if isinstance(v, tuple) else v) for k, v in case.items()},
              open(os.path.join(GOLD, 'vits_baseline0.json'), 'w'))
    print('wrote', os.path.join(GOLD, 'vits_baseline0.npz'))


if __name__ == '__main__':
    main()
