"""Multi-GPU execution of the tile path (one process per GPU, torch.distributed over NCCL/NVLink).

The reference only replicates whole images over ranks (`tools/test.py:219-229`); tiles of one image are never
sharded.  Tiles are independent given the per-image coarse outputs and the stitch is a weighted sum, so two
decompositions are offered:

* images-per-rank (bench.py `value`, weak scaling): every rank runs whole images; no data-path collective.
* tiles-per-rank (`PatchFusion.forward(..., shard=(rank, world))`, SURVEY.md §8e): the coarse branch + G2L of image b
  (whole-image kernels, ~2.7 tiles' worth of time) run on rank b % world only (`coarse_owners`), which takes
  correspondingly fewer tiles (`tile_plan`); every rank packs the coarse depth, six coarse maps and six G2L maps of
  its images into one buffer and ONE all-gather of those equal-size packs reaches every rank, while the ranks that
  own no image are already in the fine branch of their first micro-batch (the fine branch does not read coarse data).
  The tiles of all B images of a batch form one image-major list (tile i of image b is item b * n + i).  Each rank
  writes its fused predictions into a block [block_rows, ph, pw] and ONE all-gather of those blocks (5.7 MB per rank
  for one 4K P49 image) lets every rank run the deterministic stitch (pf_stitch_gather) of each image over that
  image's part of the global slot table: each canvas is bit-identical to the single-device one for any world size and
  any plan.  `model.shard_coarse = 'replicate'` keeps the variant without the pack exchange (every rank computes the
  coarse stage of every image).
"""
import torch


def coarse_owners(n_images, world, owner=0):
    """Rank that computes (and packs for everybody) the coarse branch + G2L of each image of a batch: image b on rank
    (owner + b) % world."""
    return [(owner + b) % world for b in range(n_images)]


def unpack_owned(dst, packed, world):
    """dst [B, ...] <- the all-gathered packs: packed[r] ([kmax, ...], a tensor row or list entry per rank) holds rank
    r's images r, r + world, ... (coarse_owners with owner 0) in its first rows.  One strided copy per rank."""
    B = dst.shape[0]
    for r in range(min(world, B)):
        dst[r::world].copy_(packed[r][:len(range(r, B, world))])


def tile_plan(n_items, world, owner_cost=0.0, owner=0, images=1):
    """Rank of every item of the ordered tile list.  Items are handed out one at a time to the least-loaded rank (ties:
    lowest rank); every coarse owner (`coarse_owners(images, world, owner)`) starts with `owner_cost` items' worth of
    work per image it owns - the coarse branch + G2L it computes and packs for everybody.  owner_cost = 0 is plain
    round-robin (item i -> rank i % world); images = 1 is the single-image plan (`owner` alone is charged).  A pure
    function of its arguments: every rank derives the same plan without communication."""
    load = [0.0] * world
    for r in coarse_owners(images, world, owner):
        load[r] += float(owner_cost)
    plan = []
    for _ in range(n_items):
        r = min(range(world), key=lambda q: (load[q], q))
        plan.append(r)
        load[r] += 1.0
    return plan


def shard_indices(n_items, rank, world, plan=None):
    """Items owned by `rank` (default plan: round-robin, balanced to within one item)."""
    assert 0 <= rank < world
    if plan is None:
        return list(range(rank, n_items, world))
    return [i for i in range(n_items) if plan[i] == rank]


def shard_counts(n_items, world, plan=None):
    if plan is None:
        return [len(range(r, n_items, world)) for r in range(world)]
    return [sum(1 for p in plan if p == r) for r in range(world)]


def block_rows(n_items, world, plan=None):
    """Rows of every rank's prediction block (the all-gather needs equal blocks): the largest share."""
    return max(max(shard_counts(n_items, world, plan)), 1)


def slot_table(n_items, world, plan=None):
    """Row of global item i inside the all-gathered blocks [world * block_rows, ...]: rank-major, then the item's
    position in its rank's block."""
    per = block_rows(n_items, world, plan)
    if plan is None:
        return [(i % world) * per + i // world for i in range(n_items)]
    seen = [0] * world
    out = []
    for i in range(n_items):
        out.append(plan[i] * per + seen[plan[i]])
        seen[plan[i]] += 1
    return out


def gather_blocks(block, world, group=None):
    """all_gather the per-rank prediction blocks -> [world * rows, ...] on every rank (the one collective)."""
    import torch.distributed as dist
    assert dist.get_world_size(group) == world
    block = block.contiguous()
    full = torch.empty((world * block.shape[0],) + tuple(block.shape[1:]), dtype=block.dtype, device=block.device)
    if dist.get_backend(group) == 'nccl':
        dist.all_gather_into_tensor(full, block, group=group)
    else:                                   # gloo (CPU tests): list form
        dist.all_gather(list(full.view((world,) + tuple(block.shape)).unbind(0)), block, group=group)
    return full


def stitch_reference(full, origins, slots, mask, shape):
    """torch restatement of pf_stitch_gather (CPU gloo test): fixed tile-list order, one accumulation per tile."""
    num, den = torch.zeros(shape), torch.zeros(shape)
    th, tw = mask.shape
    for (y, x), s in zip(origins, slots):
        num[y:y + th, x:x + tw] += mask * full[s]
        den[y:y + th, x:x + tw] += mask
    return num, den
