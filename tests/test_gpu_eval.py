"""Dataset evaluation on the GPU: pf_gt_prepare bit-identical to the reference's numpy branches (golden fixture from
oracle/make_golden_eval.py, and the numpy restatement on adversarial maps), pf_ingest_raw_u8 bit-identical to
float32 u8 / 255, and tools/test.py end to end equal to Tester.run fed the reference-style host preparation."""
import json
import os
import random

import numpy as np
import pytest
import torch

from patchfusion_b200 import datasets as D
from patchfusion_b200 import eval_tree as et
from patchfusion_b200 import imageio

pytestmark = [pytest.mark.gpu, pytest.mark.timeout(1800)]
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def bits_equal(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    nan = np.isnan(a) & np.isnan(b)
    return a.shape == b.shape and bool(np.all(nan | (a.view(np.int32) == b.view(np.int32))))


def _gpu(src, kind, factor=0.0, doffs=0.0, dev='cuda'):
    depth, boundary = imageio.gt_prepare(torch.from_numpy(np.ascontiguousarray(src)).to(dev), kind, factor, doffs)
    torch.cuda.synchronize()
    return depth[0, 0].cpu().numpy(), boundary[0, 0].cpu().numpy()


def test_gt_prepare_matches_reference_fixture(cuda, tmp_path):
    js, z = json.load(open(os.path.join(GOLD, 'eval_case0.json'))), np.load(os.path.join(GOLD, 'eval_case0.npz'))
    n = len(js['u4k_infos'])
    for i, info in enumerate(js['u4k_infos']):
        seed = n - int(os.path.splitext(os.path.basename(info['filename']))[0])
        depth, boundary = _gpu(et.u4k_disparity(seed), 'u4k', info['depth_factor'])
        idx = z['u4k%d_idx' % i]
        assert bits_equal(depth.reshape(-1)[idx], z['u4k%d_depth' % i]), i
        assert np.array_equal(boundary.reshape(-1)[idx].astype(np.float32), z['u4k%d_boundary' % i]), i
        img = imageio.ingest_raw(torch.from_numpy(et.u4k_frame(seed)).to(cuda))
        assert bits_equal(img[0].reshape(3, -1)[:, torch.from_numpy(idx).to(cuda)].cpu().numpy(),
                          z['u4k%d_image' % i]), i
    for kind, writer in (('mid', et.write_mid_tree), ('eth3d', et.write_eth3d_tree),
                         ('cityscapes', et.write_cityscapes_tree)):
        root = tmp_path / kind
        writer(str(root), seed=0)
        ds = D.ImageDataset(str(root / 'images'), gt_dir=str(root / 'gts'), dataset_name=kind,
                            resize_mode='depth-anything')
        src, k, factor, doffs = ds.read_ground_truth(os.path.join(str(root / 'gts'), ds.gt_files[0]))
        depth, boundary = _gpu(src, k, factor, doffs)
        idx = z['%s_idx' % kind]
        assert bits_equal(depth.reshape(-1)[idx], z['%s_depth' % kind]), kind
        assert np.array_equal(boundary.reshape(-1)[idx].astype(np.float32), z['%s_boundary' % kind]), kind


def test_metrics_on_prepared_ground_truth_match_reference(cuda):
    """pf_depth_metrics over pf_gt_prepare's depth and boundary == the reference's compute_metrics on the reference
    dataset's depth_gt (NaN depth zeroed, see oracle/make_golden_eval.py), SEE included"""
    from patchfusion_b200 import metrics as pf_metrics
    js = json.load(open(os.path.join(GOLD, 'eval_case0.json')))
    n = len(js['u4k_infos'])
    for info, want in zip(js['u4k_infos'], js['u4k_metrics']):
        seed = n - int(os.path.splitext(os.path.basename(info['filename']))[0])
        src = torch.from_numpy(et.u4k_disparity(seed)).to(cuda)
        depth, boundary = imageio.gt_prepare(src, 'u4k', info['depth_factor'])
        depth = torch.nan_to_num(depth, nan=0.0, posinf=float('inf'), neginf=float('-inf'))
        g = torch.Generator().manual_seed(7)                      # oracle fixed_prediction
        pred = (torch.rand(1, 1, 2160 // 4, 3840 // 4, generator=g) * 70 + 0.5).to(cuda)
        got = pf_metrics.compute_metrics(depth, pred, disp_gt_edges=boundary, min_depth_eval=1e-3, max_depth_eval=80)
        assert list(got) == list(want)
        for k, v in want.items():
            assert np.isfinite(v) and abs(got[k] - v) <= 1e-4 * max(1.0, abs(v)), (k, got[k], v)


def _adversarial(shape, rng, kind):
    if kind == 'cityscapes':
        x = rng.integers(0, 5, size=shape).astype(np.uint16) * rng.choice([1, 256, 257, 4000], size=shape)
        return x.astype(np.uint16)
    x = np.round(rng.uniform(-2, 6, size=shape)).astype(np.float32)      # integer steps: |delta| == 1 == th often
    x += rng.choice(np.array([0, 0, 0, 0.5, 1e-7], np.float32), size=shape)
    specials = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1.0, 2.0, 3e38, 1e-40], np.float32)
    m = rng.random(shape) < 0.2
    x[m] = rng.choice(specials, size=int(m.sum()))
    return x


@pytest.mark.parametrize('kind', ['u4k', 'mid', 'eth3d', 'cityscapes'])
def test_gt_prepare_matches_numpy_on_adversarial_maps(cuda, kind):
    rng = np.random.default_rng(11)
    factor, doffs = {'u4k': (1234.5678, 0.0), 'mid': (771535.5, 131.111), 'eth3d': (0.0, 0.0),
                     'cityscapes': (D.CITYSCAPES_FACTOR, 0.0)}[kind]
    for shape in [(1, 1), (1, 9), (9, 1), (2, 2), (7, 13), (33, 65), (257, 31), (64, 640)]:
        for rep in range(3):
            src = _adversarial(shape, rng, kind)
            want_d, want_b = D.host_ground_truth(src, kind, factor, doffs)
            got_d, got_b = _gpu(src, kind, factor, doffs)
            assert bits_equal(got_d, want_d), (kind, shape, rep)
            assert np.array_equal(got_b.astype(np.float32), want_b), (kind, shape, rep)


def test_ingest_raw_u8_all_values_and_channel_order(cuda):
    v = np.arange(256, dtype=np.uint8)
    img = np.stack([v, v[::-1], np.roll(v, 17)], 1).reshape(16, 16, 3)            # B, G, R planes differ
    out = imageio.ingest_raw(torch.from_numpy(img).to(cuda))[0].cpu().numpy()
    want = D.host_image(img).transpose(2, 0, 1)                                   # reference: float32 BGR->RGB / 255
    assert bits_equal(out, want)
    assert bits_equal(out, (img[:, :, ::-1].astype(np.float64) / 255.0).astype(np.float32).transpose(2, 0, 1))
    rgb = imageio.ingest_raw(torch.from_numpy(img).to(cuda), bgr=False)[0].cpu().numpy()
    assert bits_equal(rgb, want[::-1])


# ------------------------------------------------------------------------------------------------------- end to end
def _host_loop(conf, ckpt, cfg, mode, work_dir, dev):
    """Tester.run fed the reference-style host preparation (numpy ground truth, float32 / 255, fp32 H2D)."""
    from patchfusion_b200.config import load_config
    from patchfusion_b200.evaluate import fix_random_seed
    from patchfusion_b200.model import PatchFusion
    from patchfusion_b200.tester import Tester
    c = load_config(str(conf))
    ds = D.UnrealStereo4kDataset(**{k: v for k, v in c.val_dataloader.dataset.items() if k != 'type'})
    fix_random_seed(5621)
    model = PatchFusion(cfg)
    model.load_dict(torch.load(str(ckpt), map_location='cpu')['model_state_dict'])
    model = model.to(dev).eval()
    t = Tester(model, work_dir=str(work_dir), save=True, gray_scale=True, min_depth=ds.min_depth,
               max_depth=ds.max_depth)
    res = t.run((D.host_prepare(ds[i], dev) for i in range(len(ds))), cai_mode=mode, process_num=2,
                image_raw_shape=(2160, 3840), patch_split_num=(2, 2))
    return dict(ds.evaluate(res))


@pytest.mark.parametrize('mode', ['m1', 'r4'])
def test_cli_equals_host_prepared_loop(cuda, tmp_path, mode):
    import cv2
    from patchfusion_b200 import evaluate
    conf, ckpt, cfg = et.write_u4k_case(str(tmp_path), n_frames=2, encoder='vits', split_num=(2, 2))
    wd = tmp_path / ('cli_' + mode)
    got = evaluate.main([str(conf), '--ckp-path', str(ckpt), '--cai-mode', mode, '--test-type', 'normal', '--save',
                         '--gray-scale', '--work-dir', str(wd), '--image-raw-shape', '2160', '3840', '--patch-split-num', '2', '2'])
    assert json.load(open(wd / 'metrics.json')) == got
    assert list(got) == list(D.METRIC_KEYS)
    assert any(f.startswith('eval_cfg_vits_u4k__') and f.endswith('.log') for f in os.listdir(wd))
    random.seed(0)                                                   # the loop seeds itself, as the CLI does
    want = _host_loop(conf, ckpt, cfg, mode, tmp_path / ('host_' + mode), cuda)
    assert got == want, (got, want)
    pngs = sorted(f for f in os.listdir(tmp_path / ('host_' + mode)) if f.endswith('.png'))
    assert len(pngs) == 4 and pngs == sorted(f for f in os.listdir(wd) if f.endswith('.png'))
    for f in pngs:
        a = cv2.imread(str(wd / f), cv2.IMREAD_UNCHANGED)
        b = cv2.imread(str(tmp_path / ('host_' + mode) / f), cv2.IMREAD_UNCHANGED)
        assert a.dtype == b.dtype and np.array_equal(a, b), f
