"""Dataset evaluation, host side (no GPU): reference-format config loading, the datasets' file parsing and the numpy
restatements of the ground-truth transforms against the reference-generated fixture (tests/golden/eval_case0.*,
oracle/make_golden_eval.py), and the image-sharded metric gather over gloo."""
import json
import os

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from patchfusion_b200 import datasets as D
from patchfusion_b200 import eval_tree as et
from patchfusion_b200.config import load_config, merge_options, parse_options

pytestmark = pytest.mark.timeout(600)
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _gold():
    return json.load(open(os.path.join(GOLD, 'eval_case0.json'))), np.load(os.path.join(GOLD, 'eval_case0.npz'))


def bits_equal(a, b):
    """bit-identical, except that any two NaNs match (numpy keeps the input's NaN payload)"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    nan = np.isnan(a) & np.isnan(b)
    return a.shape == b.shape and bool(np.all(nan | (a.view(np.int32) == b.view(np.int32))))


# ------------------------------------------------------------------------------------------------------ load_config
def test_load_config_base_chain_and_options(tmp_path):
    (tmp_path / '_base_').mkdir()
    (tmp_path / '_base_' / 'data.py').write_text(
        "val_dataloader = dict(batch_size=1, num_workers=2, dataset=dict(type='A', split='a.txt', "
        "transform_cfg=dict(network_process_size=[384, 512])))\nseed = 1\nlst = [1, 2, 3]\n")
    (tmp_path / '_base_' / 'mid.py').write_text(
        "_base_ = ['./data.py']\nval_dataloader = dict(dataset=dict(resize_mode='zoe'))\nlst = [9]\n")
    (tmp_path / 'cfg.py').write_text(
        "_base_ = ['_base_/mid.py']\nmin_depth = 1e-3\nmodel = dict(type='PatchFusion', config=dict(min_depth=min_depth,"
        " shape=(2160, 3840)))\nval_dataloader = dict(dataset=dict(resize_mode='depth-anything', "
        "transform_cfg=dict(network_process_size=[392, 518])))\n")
    cfg = load_config(str(tmp_path / 'cfg.py'))
    ds = cfg.val_dataloader.dataset
    assert (ds.type, ds.split, ds.resize_mode) == ('A', 'a.txt', 'depth-anything')
    assert ds.transform_cfg.network_process_size == [392, 518]
    assert cfg.val_dataloader.num_workers == 2 and cfg.seed == 1 and cfg.lst == [9]      # lists replace
    assert cfg.model.config.shape == (2160, 3840) and cfg.model.config.min_depth == 1e-3
    opts = parse_options(['val_dataloader.dataset.split=b.txt', 'seed=7', 'x.y=[1,2]', 'x.t=(1,2)', 'x.c=a,b',
                          'x.b=false', 'x.n=None', 'x.f=0.5', "x.s='q'"])
    merge_options(cfg, opts)
    assert cfg.val_dataloader.dataset.split == 'b.txt' and cfg.val_dataloader.dataset.type == 'A'
    assert cfg.seed == 7
    assert (cfg.x.y, cfg.x.t, cfg.x.c, cfg.x.b, cfg.x.n, cfg.x.f, cfg.x.s) == ([1, 2], (1, 2), ['a', 'b'], False,
                                                                               None, 0.5, 'q')


# ---------------------------------------------------------------------------------------------------------- datasets
def test_u4k_split_extrinsics_sorting_basenames(tmp_path):
    js, _ = _gold()
    split = et.write_u4k_tree(str(tmp_path), len(js['u4k_infos']), seed=0)
    assert open(split).read() == js['u4k_split']
    ds = D.UnrealStereo4kDataset('infer', str(tmp_path), split, {'network_process_size': [392, 518]}, 1e-3, 80,
                                 resize_mode='depth-anything')
    assert len(ds) == len(js['u4k_infos'])
    for info, want, base in zip(ds.data_infos, js['u4k_infos'], js['u4k_basenames']):
        assert os.path.relpath(info['img_path'], str(tmp_path)) == want['img_path']
        assert os.path.relpath(info['depth_map_path'], str(tmp_path)) == want['depth_map_path']
        assert info['filename'] == want['filename']
        assert info['focal'] == want['focal'] and info['depth_factor'] == want['depth_factor']
        assert ds.basename(info['filename']) == base
    s = ds[0]
    assert s['image'].shape == (2160, 3840, 3) and s['image'].dtype == np.uint8 and s['gt'].dtype == np.float32
    assert s['img_file_basename'] == js['u4k_basenames'][0] and s['image_resize'] is None


def test_dataset_rejections(tmp_path):
    with pytest.raises(NotImplementedError):
        D.UnrealStereo4kDataset('train', str(tmp_path), None, {}, 1e-3, 80, resize_mode='depth-anything')
    split = et.write_u4k_tree(str(tmp_path), 1)
    with pytest.raises(NotImplementedError):
        D.UnrealStereo4kDataset('infer', str(tmp_path), split, {}, 1e-3, 80)            # default resize_mode 'zoe'
    (tmp_path / 'img').mkdir()
    (tmp_path / 'gt').mkdir()
    (tmp_path / 'img' / 'a.png').write_bytes(b'')
    (tmp_path / 'gt' / 'a.exr').write_bytes(b'')
    ds = D.ImageDataset(str(tmp_path / 'img'), gt_dir=str(tmp_path / 'gt'), dataset_name='gta',
                        resize_mode='depth-anything')
    with pytest.raises(NotImplementedError, match='imageio'):
        ds.read_ground_truth(str(tmp_path / 'gt' / 'a.exr'))


def test_image_dataset_pairs_sorted_files(tmp_path):
    et.write_mid_tree(str(tmp_path), seed=0)
    ds = D.ImageDataset(str(tmp_path / 'images'), gt_dir=str(tmp_path / 'gts'), dataset_name='mid',
                        image_resolution=[64, 96], resize_mode='depth-anything')
    s = ds[0]
    assert s['img_file_basename'] == 'mid0' and s['image_resize'] == (64, 96) and s['gt_kind'] == 'mid'
    assert s['factor'] == 193.001 * 3997.684 and s['doffs'] == 131.111
    assert bits_equal(s['gt'], et.mid_disparity(0))
    assert D.ImageDataset.image_name('x.jpeg') == 'x' and D.ImageDataset.image_name('y.jpg') == 'y'


# ------------------------------------------------------------------------------------ ground-truth transforms (numpy)
def _u4k_sources(js):
    n = len(js['u4k_infos'])
    for i, info in enumerate(js['u4k_infos']):
        seed = n - int(os.path.splitext(os.path.basename(info['filename']))[0])   # file k holds seed n - k
        yield i, seed, info['depth_factor']


def test_host_u4k_matches_reference_fixture():
    js, z = _gold()
    for i, seed, factor in _u4k_sources(js):
        depth, boundary = D.host_ground_truth(et.u4k_disparity(seed), 'u4k', factor)
        idx = z['u4k%d_idx' % i]
        assert bits_equal(depth.reshape(-1)[idx], z['u4k%d_depth' % i])
        assert np.array_equal(boundary.reshape(-1)[idx], z['u4k%d_boundary' % i])
        img = D.host_image(et.u4k_frame(seed)).transpose(2, 0, 1).reshape(3, -1)[:, idx]
        assert bits_equal(img, z['u4k%d_image' % i])
    # the float32-rounded-constant form the kernel uses
    d = et.u4k_disparity(0)
    with np.errstate(divide='ignore'):
        assert bits_equal(D.host_ground_truth(d, 'u4k', 1234.5678)[0], np.float32(1234.5678) / d)


@pytest.mark.parametrize('kind', ['mid', 'eth3d', 'cityscapes'])
def test_host_general_matches_reference_fixture(kind, tmp_path):
    js, z = _gold()
    writer = {'mid': et.write_mid_tree, 'eth3d': et.write_eth3d_tree, 'cityscapes': et.write_cityscapes_tree}[kind]
    writer(str(tmp_path), seed=0)
    ds = D.ImageDataset(str(tmp_path / 'images'), gt_dir=str(tmp_path / 'gts'), dataset_name=kind,
                        resize_mode='depth-anything')
    src, k, factor, doffs = ds.read_ground_truth(os.path.join(str(tmp_path / 'gts'), ds.gt_files[0]))
    assert k == kind and list(src.shape) == js['%s_shape' % kind]
    depth, boundary = D.host_ground_truth(src, kind, factor, doffs)
    idx = z['%s_idx' % kind]
    assert bits_equal(depth.reshape(-1)[idx], z['%s_depth' % kind])
    assert np.array_equal(boundary.reshape(-1)[idx], z['%s_boundary' % kind])


def test_evaluate_reference_order():
    r = [dict(zip(D.METRIC_KEYS, np.arange(10.0) + j)) for j in range(3)]
    r[1]['rmse'] = float('nan')
    out = D.UnrealStereo4kDataset.evaluate(r)
    assert list(out) == ['a1', 'a2', 'a3', 'abs_rel', 'rmse', 'log_10', 'rmse_log', 'silog', 'sq_rel', 'see']
    assert out['a1'] == 1.0 and out['rmse'] == 5.0 and out['see'] == 10.0


def test_header_gt_kinds_match_imageio():
    import re
    from patchfusion_b200 import imageio
    hdr = open(os.path.join(os.path.dirname(GOLD), '..', 'include', 'pf_b200.h')).read()
    kinds = {k.lower(): int(v) for k, v in re.findall(r'#define\s+PF_GT_([A-Z0-9]+)\s+(\d+)', hdr)}
    assert kinds == imageio.GT_KINDS


# -------------------------------------------------------------------------------------------- image-sharded gather
class _StubDataset:
    """n images whose 'metrics' are a function of the index; records which indices were read and prepared"""

    def __init__(self, n, log):
        self.n, self.log = n, log

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        self.log.append(('read', i))
        return dict(index=i)

    def prepare(self, s, device):
        self.log.append(('prepare', s['index']))
        return s


class _StubTester:
    @staticmethod
    def metrics(i):
        r = {k: float(np.float64(i) * 1.1 + j / 7.0) for j, k in enumerate(D.METRIC_KEYS)}
        if i % 3 == 2:
            r['rmse'] = float('nan')
        return r

    def run(self, samples, **kw):
        return [self.metrics(s['index']) for s in samples]


class _RandomStubTester(_StubTester):
    """draws from `random` per image, as rN random tiles do"""

    def run(self, samples, **kw):
        import random
        return [dict(_StubTester.metrics(s['index']), a1=random.random()) for s in samples]


def _same(a, b):
    """equal metric lists: same keys in the same order, equal values, NaN where NaN"""
    return len(a) == len(b) and all(list(x) == list(y) and np.array_equal(list(x.values()), list(y.values()),
                                                                          equal_nan=True) for x, y in zip(a, b))


def _shard_worker(rank, world, port, n, out):
    from patchfusion_b200 import evaluate as E
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    log = []
    got = E.run_images(_StubTester(), _StubDataset(n, log), torch.device('cpu'), rank, world, num_workers=2)
    E.fix_random_seed(5621)                                   # every rank seeds itself (evaluate.main)
    drawn = E.run_images(_RandomStubTester(), _StubDataset(n, []), torch.device('cpu'), rank, world)
    out.put((rank, got, log, drawn))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize('world,n', [(2, 7), (3, 7), (3, 2)])
def test_gloo_image_shard_gather_equals_single_process(world, n):
    from patchfusion_b200 import evaluate as E
    single_log = []
    single = E.run_images(_StubTester(), _StubDataset(n, single_log), torch.device('cpu'), 0, 1)
    assert _same(single, [_StubTester.metrics(i) for i in range(n)])
    ctx = mp.get_context('spawn')
    out = ctx.Queue()
    port = 29500 + (os.getpid() * 7 + world) % 3000
    procs = [ctx.Process(target=_shard_worker, args=(r, world, port, n, out)) for r in range(world)]
    for p in procs:
        p.start()
    res = [out.get(timeout=240) for _ in range(world)]
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    computed = []
    want_drawn = E.shard_reference(_RandomStubTester(), _StubDataset(n, []), torch.device('cpu'), world, 5621)
    for rank, got, log, drawn in res:
        assert _same(got, single)
        assert _same(drawn, want_drawn)              # random draws restart per rank: the shard-reseeded reference
        mine = [i for tag, i in log if tag == 'prepare']
        assert mine == list(range(rank, n, world))                   # in order, no padded duplicate
        computed += mine
    assert sorted(computed) == list(range(n))


def test_metric_rows_round_trip():
    from patchfusion_b200 import evaluate as E
    n, world = 5, 2
    res = [_StubTester.metrics(i) for i in range(n)]
    del res[4]['see']
    rows = np.stack([E.metric_rows(res[r::world], n, world) for r in range(world)])
    assert rows.shape == (2, 3, 12) and rows[1, 2, 0] == 0.0             # rank 1's padding row: not computed
    back = E.interleave_rows(rows, n)
    assert _same(back, res)


class _FailingDataset(_StubDataset):
    def __getitem__(self, i):
        if i >= 2:
            raise OSError('unreadable image %d' % i)
        return dict(index=i)


def test_prepared_samples_reader_errors():
    """a reader error reaches the consumer; a consumer that stops early never waits on a reader stuck on a full queue"""
    import time
    it = iter(D.PreparedSamples(_FailingDataset(6, []), range(6), 'cpu', num_workers=1, pin_memory=False))
    assert next(it)['index'] == 0 and next(it)['index'] == 1
    with pytest.raises(OSError, match='unreadable image 2'):
        next(it)
    it = iter(D.PreparedSamples(_FailingDataset(6, []), range(6), 'cpu', num_workers=1, pin_memory=False))
    next(it)
    time.sleep(0.3)                       # the reader has queued image 1 and failed on image 2 against a full queue
    t = time.time()
    it.close()
    assert time.time() - t < 5
