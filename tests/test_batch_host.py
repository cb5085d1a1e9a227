"""Host logic of the batched forward (no GPU): the image-major tile list, each image's part of the slot table, the
coarse-owner plan, the random draws of a batch, and - under a gloo world of 2 - the all-gather of coarse packs and
prediction blocks followed by per-image stitches, which must reproduce every single-image canvas bit for bit."""
import os
import random

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from patchfusion_b200.model import TiledModel
from patchfusion_b200.parallel import (block_rows, coarse_owners, gather_blocks, shard_counts, shard_indices,
                                       slot_table, stitch_reference, tile_plan, unpack_owned)

pytestmark = pytest.mark.timeout(300)

RAW = [(0, 0), (0, 32), (24, 0), (24, 32), (12, 16)]        # one image's tile list (5 tiles)


def test_tile_list_is_image_major():
    for B in (1, 2, 5):
        tiles = TiledModel.batch_tiles(RAW, B)
        assert len(tiles) == B * len(RAW)
        for b in range(B):
            assert tiles[b * len(RAW):(b + 1) * len(RAW)] == [(b, y, x) for (y, x) in RAW]
        assert TiledModel.image_ranges(tiles, B) == [(b * len(RAW), (b + 1) * len(RAW)) for b in range(B)]
        yx, img = TiledModel.split_tiles(tiles)
        assert yx == RAW * B and img == [b for b in range(B) for _ in RAW]
    assert TiledModel.split_tiles(RAW) == (RAW, [0] * len(RAW))       # single-image callers pass (y, x)
    # a random-phase chunk may start or end inside an image, or miss one entirely
    part = [(1, 3, 4), (1, 5, 6), (3, 0, 0)]
    assert TiledModel.image_ranges(part, 4) == [(0, 0), (0, 2), (2, 2), (2, 3)]


@pytest.mark.parametrize('B', [1, 2, 5])
@pytest.mark.parametrize('W', [1, 2, 3, 8])
def test_per_image_slot_tables(B, W):
    """every plan (round-robin, coarse-owner) puts every tile of every image in exactly one rank's block, and image b's
    part of the slot table addresses exactly the rows its tiles were written to"""
    n = len(RAW)
    N = B * n                                                # W = 8 > B and > the tiles of one image
    for plan in (None, tile_plan(N, W, 2.7, images=B)):
        owned = [shard_indices(N, r, W, plan) for r in range(W)]
        assert sorted(i for o in owned for i in o) == list(range(N))
        per = block_rows(N, W, plan)
        slots = slot_table(N, W, plan)
        assert len(set(slots)) == N and max(slots) < W * per
        row_of = {}
        for r in range(W):
            for j, i in enumerate(owned[r]):
                row_of[i] = r * per + j
        for b in range(B):
            sub = slots[b * n:(b + 1) * n]
            assert sub == [row_of[b * n + i] for i in range(n)]


def test_coarse_owner_plan():
    for B, W in [(1, 1), (1, 8), (2, 2), (2, 3), (5, 2), (5, 3), (5, 8), (8, 8), (4, 8)]:
        owners = coarse_owners(B, W)
        assert owners == [b % W for b in range(B)]
        N = 49 * B
        plan = tile_plan(N, W, 2.7, images=B)
        counts = shard_counts(N, W, plan)
        assert sum(counts) == N
        # the load (tiles + 2.7 per owned image) is balanced to within one tile
        load = [counts[r] + 2.7 * owners.count(r) for r in range(W)]
        assert max(load) - min(load) <= 1.0 + 1e-9, (B, W, load)
    # 4 images on 8 ranks: ranks 0-3 each own one coarse stage and take fewer tiles than ranks 4-7
    c = shard_counts(4 * 49, 8, tile_plan(4 * 49, 8, 2.7, images=4))
    assert min(c[4:]) > max(c[:4])
    # W > number of tiles: some ranks get nothing, nothing is lost
    plan = tile_plan(2, 8, 2.7, images=1)
    assert sorted(plan) == plan and 0 not in plan and len(plan) == 2


def test_tile_plan_single_image_unchanged():
    """images=1 (the default) is the plan of the single-image forward, as before batching"""
    for n, w, c in [(49, 8, 2.7), (49, 2, 2.7), (353, 8, 2.7), (5, 8, 2.7), (16, 4, 100.0), (49, 8, 0.0)]:
        assert tile_plan(n, w, c) == tile_plan(n, w, c, images=1)
    assert shard_counts(49, 8, tile_plan(49, 8, owner_cost=2.7)) == [4, 7, 7, 7, 6, 6, 6, 6]
    assert shard_counts(49, 2, tile_plan(49, 2, 2.7)) == [23, 26]
    assert tile_plan(10, 4) == [i % 4 for i in range(10)]


@pytest.mark.parametrize('B', [1, 2, 5])
def test_random_draws_match_sequential_calls(B):
    H, W, h, w, pn, calls = 1080, 1920, 540, 960, 3, 4
    random.seed(123)
    seq = []
    for b in range(B):
        one = TiledModel._draw_random_boxes(None, calls, pn, H, W, h, w, None, None, 'cpu')
        seq += [(b,) + t[1:] for t in one]
        assert all(t[0] == 0 for t in one)
    after_seq = random.random()
    random.seed(123)
    batch = TiledModel._draw_random_boxes(None, calls, pn, H, W, h, w, None, None, 'cpu', B)
    assert batch == seq and random.random() == after_seq       # same draws, same state afterwards
    assert TiledModel.image_ranges(batch, B) == [(b * calls * pn, (b + 1) * calls * pn) for b in range(B)]


def test_unpack_owned():
    for B, W in [(1, 1), (1, 3), (3, 2), (5, 2), (5, 8), (4, 4)]:
        kmax = -(-B // W)
        full = torch.arange(B * 6, dtype=torch.float32).view(B, 2, 3)
        packed = torch.full((W, kmax, 2, 3), float('nan'))
        for b, r in enumerate(coarse_owners(B, W)):
            packed[r, b // W] = full[b]
        dst = torch.full_like(full, float('nan'))
        unpack_owned(dst, packed, W)
        assert torch.equal(dst, full)


def _worker(rank, world, port, out):
    from patchfusion_b200.model import PatchFusion
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    g = torch.Generator().manual_seed(0)
    th, tw, shape = 24, 32, (48, 64)
    n = len(RAW)
    same = True
    for B in (1, 2, 3):
        preds = torch.rand(B, n, th, tw, generator=g)            # every image's fused tiles
        coarse = torch.rand(B, 7, 5, generator=g)                # stands in for one item of the coarse pack
        mask = torch.rand(th, tw, generator=g) + 1e-3
        want = [stitch_reference(preds[b], RAW, list(range(n)), mask, shape) for b in range(B)]
        # coarse packs: rank r packs its images into a kmax-row pack; one all-gather; unpack into batch order
        kmax = -(-B // world)
        mine = [b for b, o in enumerate(coarse_owners(B, world)) if o == rank]
        pack = torch.full((kmax, 7, 5), float('nan'))
        for j, b in enumerate(mine):
            pack[j] = coarse[b]
        gathered = torch.empty((world, kmax * 35))
        PatchFusion._gather_packs(pack.view(-1), gathered, None)
        batch = torch.full_like(coarse, float('nan'))
        unpack_owned(batch, gathered.view(world, kmax, 7, 5), world)
        same = same and torch.equal(batch, coarse)
        # prediction blocks of the image-major tile list, per-image stitch over that image's slot sub-table
        N = B * n
        for plan in (None, tile_plan(N, world, 2.7, images=B)):
            own = shard_indices(N, rank, world, plan)
            per = block_rows(N, world, plan)
            block = torch.full((per, th, tw), float('nan'))       # padding rows must never be read
            for j, i in enumerate(own):
                block[j] = preds[i // n, i % n]
            full = gather_blocks(block, world)
            slots = slot_table(N, world, plan)
            for b in range(B):
                num, den = stitch_reference(full, RAW, slots[b * n:(b + 1) * n], mask, shape)
                same = same and torch.equal(num, want[b][0]) and torch.equal(den, want[b][1])
    if rank == 0:
        out.put(same)
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_batch_gather_matches_per_image_runs():
    ctx = mp.get_context('spawn')
    out = ctx.Queue()
    port = 31500 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    assert out.get(timeout=5) is True
