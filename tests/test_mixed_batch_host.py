"""Host logic of the mixed-geometry batch (no GPU): images with their own tile_cfg and cai_mode in one forward.  The
tile list, ROI boxes, slot tables and random draws of a mixed batch must be the concatenation of the single-image ones;
a gloo world of 2 must stitch every image of a mixed batch as the single-image stitch does; bad input raises; and
pf_crop_resize_multi and its descriptor are bound as include/pf_b200.h declares them."""
import ctypes
import os
import random
import re
import subprocess

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from patchfusion_b200.model import TiledModel
from patchfusion_b200.parallel import (block_rows, gather_blocks, shard_indices, slot_table, stitch_reference,
                                       tile_plan)

pytestmark = pytest.mark.timeout(300)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = os.path.join(ROOT, 'include', 'pf_b200.h')
PPS = (392, 518)
# (image_raw_shape, patch_split_num, cai_mode): uneven tile counts (4, 21, 9 + random, 1, 49 + random)
MIX = [((1080, 1920), (2, 2), 'm1'), ((720, 1280), (2, 4), 'm2'), ((1080, 1920), (2, 2), 'r4'),
       ((540, 960), (1, 1), 'm1'), ((2160, 3840), (4, 4), 'r9')]


class _Host:
    """the parts of TiledModel that need no device and no weights"""
    patch_process_shape = PPS
    tile_cfg = None
    prepare_tile_cfg = TiledModel.prepare_tile_cfg
    _batch_inputs = TiledModel._batch_inputs


def _cfg(shape, split):
    return _Host().prepare_tile_cfg(shape, split)


def _single_tiles(shape, split, mode):
    """the reference's regular tiles of one image (baseline_pretrain.py:221-251), restated: (raw, proc) origins"""
    H, W = shape
    h, w = H // split[0], W // split[1]
    ph, pw = PPS
    passes = [(0, 0, 0, 0)]
    if mode == 'm2' or mode.startswith('r'):
        passes += [(0, w // 2, 0, pw // 2), (h // 2, 0, ph // 2, 0), (h // 2, w // 2, ph // 2, pw // 2)]
    raw, proc = [], []
    for oy, ox, py, px in passes:
        for a in range((H - oy) // h):
            for b in range((W - ox) // w):
                raw.append((h * a + oy, w * b + ox))
                proc.append((ph * a + py, pw * b + px))
    return raw, proc


def _single_boxes(raw, shape, split):
    """the single-image forward's boxes: int pixel box * fp32 factor of the image (baseline_pretrain.py:268-282)"""
    H, W = shape
    h, w = H // split[0], W // split[1]
    fx, fy = np.float32(1 / W * PPS[1]), np.float32(1 / H * PPS[0])
    return np.array([[np.float32(x) * fx, np.float32(y) * fy, np.float32(x + w) * fx, np.float32(y + h) * fy]
                     for (y, x) in raw], dtype=np.float32)


def _geom(shape, split):
    return tuple(shape) + (shape[0] // split[0], shape[1] // split[1]) + PPS


def test_tiles_and_boxes_are_the_single_image_ones():
    per = [TiledModel.regular_tiles(_cfg(s, p), m, PPS) for s, p, m in MIX]
    for (s, p, m), (raw, proc) in zip(MIX, per):
        assert (raw, proc) == _single_tiles(s, p, m)
    tiles = TiledModel.mixed_tiles([r for r, _ in per])
    ranges = TiledModel.image_ranges(tiles, len(MIX))
    assert [b - a for a, b in ranges] == [4, 21, 9, 1, 49]
    for b, ((s, p, m), (raw, _)) in enumerate(zip(MIX, per)):
        i0, i1 = ranges[b]
        assert tiles[i0:i1] == [(b, y, x) for (y, x) in raw]
    boxes = TiledModel.roi_boxes(tiles, [_geom(s, p) for s, p, _ in MIX])
    assert boxes.dtype == np.float32
    want = np.concatenate([_single_boxes(raw, s, p) for (s, p, _), (raw, _) in zip(MIX, per)])
    assert boxes.tobytes() == want.tobytes()                                   # bit for bit
    # a batch of one geometry is the old image-major list, and (y, x) items are image 0's
    raw0 = per[1][0]
    assert TiledModel.mixed_tiles([raw0] * 3) == TiledModel.batch_tiles(raw0, 3)
    assert TiledModel.roi_boxes(raw0, [_geom(*MIX[1][:2])]).tobytes() == _single_boxes(raw0, *MIX[1][:2]).tobytes()


@pytest.mark.parametrize('W', [1, 2, 3, 8])
def test_mixed_slot_tables(W):
    """every plan puts each tile of each image in one rank's block, and image b's part of the slot table addresses
    the rows its tiles were written to, in the image's own tile order"""
    tiles = TiledModel.mixed_tiles([TiledModel.regular_tiles(_cfg(s, p), m, PPS)[0] for s, p, m in MIX])
    N, B = len(tiles), len(MIX)
    for plan in (None, tile_plan(N, W, 2.7, images=B)):
        per = block_rows(N, W, plan)
        gathered = [None] * (W * per)
        for r in range(W):
            for j, i in enumerate(shard_indices(N, r, W, plan)):
                gathered[r * per + j] = tiles[i]
        slots = slot_table(N, W, plan)
        for b, (i0, i1) in enumerate(TiledModel.image_ranges(tiles, B)):
            assert [gathered[s] for s in slots[i0:i1]] == tiles[i0:i1]
            assert all(t[0] == b for t in tiles[i0:i1])


@pytest.mark.parametrize('rule', ['patchfusion', 'baseline'])
def test_random_draws_match_sequential_calls(rule):
    pn = 3
    calls = (lambda m: int(m[1:]) // pn) if rule == 'patchfusion' else (lambda m: int(m[1:]))
    specs = [((calls(m) if m[0] == 'r' else 0),) + _geom(s, p)[:4] for s, p, m in MIX]
    random.seed(77)
    seq = []
    for b, sp in enumerate(specs):
        one = TiledModel.draw_random_boxes([sp], pn, None, None, 'cpu')
        assert all(t[0] == 0 for t in one)
        seq += [(b,) + t[1:] for t in one]
    after = random.random()
    random.seed(77)
    got = TiledModel.draw_random_boxes(specs, pn, None, None, 'cpu')
    assert got == seq and random.random() == after
    counts = [b - a for a, b in TiledModel.image_ranges(got, len(MIX))]
    assert counts == [sp[0] * pn for sp in specs] and counts[2] > 0 and counts[4] > 0 and counts[0] == 0


def _worker(rank, world, port, out):
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    g = torch.Generator().manual_seed(0)
    th, tw = 8, 12                                           # predictions at a small stand-in for patch_process_shape
    mix = [((12, 16), (2, 2), 'm2'), ((6, 8), (1, 1), 'm1'), ((12, 32), (2, 4), 'm1')]
    cfgs = []
    for shape, split, mode in mix:
        c = {'image_raw_shape': shape, 'patch_split_num': split, 'patch_raw_shape': (shape[0] // split[0],
             shape[1] // split[1]), 'patch_reensemble_shape': (th * split[0], tw * split[1])}
        cfgs.append(c)
    per = [TiledModel.regular_tiles(c, m, (th, tw)) for c, (_, _, m) in zip(cfgs, mix)]
    tiles = TiledModel.mixed_tiles([r for r, _ in per])
    N, B = len(tiles), len(mix)
    preds = torch.rand(N, th, tw, generator=g)
    mask = torch.rand(th, tw, generator=g) + 1e-3
    ranges = TiledModel.image_ranges(tiles, B)
    want = [stitch_reference(preds[i0:i1], per[b][1], list(range(i1 - i0)), mask, cfgs[b]['patch_reensemble_shape'])
            for b, (i0, i1) in enumerate(ranges)]
    same = True
    for plan in (None, tile_plan(N, world, 2.7, images=B)):
        own = shard_indices(N, rank, world, plan)
        block = torch.full((block_rows(N, world, plan), th, tw), float('nan'))   # padding rows must never be read
        for j, i in enumerate(own):
            block[j] = preds[i]
        full = gather_blocks(block, world)
        slots = slot_table(N, world, plan)
        for b, (i0, i1) in enumerate(ranges):
            num, den = stitch_reference(full, per[b][1], slots[i0:i1], mask, cfgs[b]['patch_reensemble_shape'])
            same = same and torch.equal(num, want[b][0]) and torch.equal(den, want[b][1])
    if rank == 0:
        out.put(same)
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_mixed_stitch_matches_per_image():
    ctx = mp.get_context('spawn')
    out = ctx.Queue()
    port = 33600 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    assert out.get(timeout=5) is True


# ---------------------------------------------------------------------------------------------------- input checks
def test_batch_inputs():
    h = _Host()
    a, b = torch.zeros(1, 3, 1080, 1920), torch.zeros(1, 3, 720, 1280)
    c1, c2 = {'image_raw_shape': [1080, 1920], 'patch_split_num': [2, 2]}, {'image_raw_shape': (720, 1280),
                                                                           'patch_split_num': (2, 4)}
    imgs, cfgs, modes, mixed = h._batch_inputs([a, b], [c1, c2], 'm1')
    assert mixed and imgs[0] is a and imgs[1] is b and modes == ['m1', 'm1'] and cfgs[1]['patch_raw_shape'] == (360, 320)
    # one geometry: the tensor path, unchanged
    x, cfg, mode, mixed = h._batch_inputs(torch.zeros(2, 3, 1080, 1920), c1, 'm2')
    assert not mixed and x.shape[0] == 2 and cfg['patch_raw_shape'] == (540, 960) and mode == 'm2'
    # a list that shares one geometry and mode comes back as the tensor batch
    x, cfg, mode, mixed = h._batch_inputs([a, a + 1], [c1, dict(c1)], ['r4', 'r4'])
    assert mixed and torch.equal(x, torch.cat([a, a + 1])) and mode == 'r4'
    # per-image modes with one tensor batch
    imgs, _, modes, mixed = h._batch_inputs(torch.zeros(2, 3, 1080, 1920), c1, ['m1', 'm2'])
    assert mixed and len(imgs) == 2 and imgs[0].shape == (1, 3, 1080, 1920) and modes == ['m1', 'm2']


def test_bad_input_raises():
    h = _Host()
    a, b = torch.zeros(1, 3, 1080, 1920), torch.zeros(1, 3, 720, 1280)
    c1, c2 = {'image_raw_shape': [1080, 1920], 'patch_split_num': [2, 2]}, {'image_raw_shape': [720, 1280],
                                                                           'patch_split_num': [2, 4]}
    with pytest.raises(ValueError, match='tile_cfg'):
        h._batch_inputs([a, b], [c1], 'm1')
    with pytest.raises(ValueError, match='cai_mode'):
        h._batch_inputs([a, b], [c1, c2], ['m1'])
    with pytest.raises(AssertionError, match='divisible'):
        h._batch_inputs([a, b], [c1, {'image_raw_shape': [720, 1280], 'patch_split_num': [7, 4]}], 'm1')
    with pytest.raises(AssertionError, match='image_raw_shape'):
        h._batch_inputs([b, a], [c1, c2], 'm1')


def test_forward_checks_before_any_device_work():
    """PatchFusion.forward raises on a bad mixed batch before it needs the engine (so on a CPU model too)"""
    from patchfusion_b200.configs import depth_anything_patchfusion
    from patchfusion_b200.model import PatchFusion
    model = PatchFusion(depth_anything_patchfusion('vits'))
    a, b = torch.zeros(1, 3, 1080, 1920), torch.zeros(1, 3, 720, 1280)
    lr = torch.zeros(2, 3, *PPS)
    c1, c2 = {'image_raw_shape': [1080, 1920], 'patch_split_num': [2, 2]}, {'image_raw_shape': [720, 1280],
                                                                           'patch_split_num': [2, 4]}
    with pytest.raises(ValueError):
        model(mode='infer', image_lr=lr, image_hr=[a, b], tile_cfg=[c1, c2, c2])
    with pytest.raises(AssertionError):
        model(mode='infer', image_lr=lr[:1], image_hr=[a, b], tile_cfg=[c1, c2])
    with pytest.raises(AssertionError):
        model(mode='infer', image_lr=lr, image_hr=[a, b], tile_cfg=[c1, {'image_raw_shape': [721, 1280],
                                                                         'patch_split_num': [2, 4]}])
    with pytest.raises(AssertionError):
        model(mode='infer', image_lr=lr, image_hr=[a, b], tile_cfg=[c2, c1])


def test_baseline_coarse_target_rejects_a_list():
    from patchfusion_b200.baseline import BaselinePretrain
    from test_baseline_host import pretrain_model_cfg
    cfg = pretrain_model_cfg('vits', 'coarse')
    cfg.pop('type')
    with pytest.raises(ValueError, match='coarse target'):
        BaselinePretrain(**cfg)(mode='infer', image_lr=[torch.zeros(1, 3, 378, 518)], image_hr=None)


# ---------------------------------------------------------------------------------------------------- C ABI
def test_crop_resize_multi_export_and_arity():
    from patchfusion_b200 import build, lib
    path = build.build()
    out = subprocess.check_output(['nm', '-D', '--defined-only', path], text=True)
    assert 'pf_crop_resize_multi' in set(l.split()[-1] for l in out.splitlines() if l.strip())
    src = re.sub(r'/\*.*?\*/', '', open(HDR).read(), flags=re.S)
    args = re.search(r'\bint\s+pf_crop_resize_multi\s*\(([^;{]*?)\)\s*;', src, flags=re.S).group(1)
    assert len(args.split(',')) == len(lib.SIGNATURES['pf_crop_resize_multi']) == 8
    assert 'pf_crop_resize_batched' in lib.SIGNATURES and 'pf_crop_resize' in lib.SIGNATURES
    assert lib.load().pf_crop_resize_multi.argtypes is not None


def test_crop_image_layout(tmp_path):
    from patchfusion_b200.lib import CropImage
    prog = '#include <stdio.h>\n#include <stddef.h>\n#include "%s"\nint main(){' % HDR
    prog += 'printf("sizeof %zu\\n", sizeof(pf_crop_image));'
    for f in CropImage._fields_:
        prog += 'printf("%s %%zu\\n", offsetof(pf_crop_image, %s));' % (f[0], f[0])
    prog += 'return 0;}'
    c = tmp_path / 'crop.c'
    c.write_text(prog)
    exe = tmp_path / 'crop'
    subprocess.check_call(['gcc', str(c), '-o', str(exe)])
    seen = 0
    for line in subprocess.check_output([str(exe)], text=True).splitlines():
        k, v = line.split()
        assert (ctypes.sizeof(CropImage) if k == 'sizeof' else getattr(CropImage, k).offset) == int(v), k
        seen += 1
    assert seen == 1 + len(CropImage._fields_)
