"""Drop-in `BaselinePretrain` for the reference's `estimator.models.baseline_pretrain.BaselinePretrain` (inference
path): one ZoeDepth / Depth-Anything branch, the paper's two baselines.

    target='coarse'   one branch forward over a batch of whole low-resolution images (BP:365-367, 419)
    target='fine'     the same network on every tile of a high-resolution image, blended with the Gaussian running
                      average of `PatchFusion` but without guided fusion (BP:369-414)

Same constructor, `state_dict()` key layout (only the built branch), `load_dict` / `get_save_dict` (the branch-only
files `PatchFusion(load_branch=True)` reads back) and error behaviour as the reference; the arithmetic runs on
libpf_b200 (sm_90a) through `Engine(parts=(branch,))`.  There is no CPU path: calling forward on a CPU model raises.

Two reference behaviours differ from `PatchFusion` and are kept: rN runs N `random_tile` calls of process_num tiles
each (BP:407-410; PatchFusion runs N // process_num), and the fine target returns an empty info dict (BP:412-414).
"""
import torch
import torch.nn as nn

from .model import AttrDict, Resize, TiledModel
from .params import _get, branch_layout, synthetic_state_dict


def _attr(cfg):
    if not isinstance(cfg, dict) and hasattr(cfg, 'to_dict'):
        cfg = cfg.to_dict()
    return AttrDict(dict(cfg))


class BaselinePretrain(TiledModel):
    def __init__(self, coarse_branch, fine_branch, sigloss, min_depth, max_depth, image_raw_shape=(2160, 3840),
                 patch_process_shape=(384, 512), patch_split_num=(4, 4), target='coarse', coarse_branch_zoe=None):
        nn.Module.__init__(self)
        # patch_process_shape is deliberately not checked against the 14-px patch here: the shipped coarse configs
        # keep the (384, 512) default, and the reference fails only when a forward runs at a non-multiple of 14
        self.patch_process_shape = tuple(patch_process_shape)
        self.tile_cfg = self.prepare_tile_cfg(image_raw_shape, patch_split_num)
        self.min_depth = min_depth
        self.max_depth = max_depth
        self.coarse_branch_cfg = _attr(coarse_branch)
        self.fine_branch_cfg = _attr(fine_branch)
        self.sigloss_cfg = sigloss          # SILogLoss has no parameters and only serves mode='train'
        self.target = target
        self.branch = None                  # 'coarse' | 'fine': the one branch this model holds
        if target in ('coarse', 'fine'):
            cfg = self.coarse_branch_cfg if target == 'coarse' else self.fine_branch_cfg
            if cfg.type == 'ZoeDepth':
                raise NotImplementedError(
                    "branch type 'ZoeDepth' (BEiT-L backbone from an un-vendored torch.hub repo) is not built; "
                    "use 'DA-ZoeDepth'")
            if cfg.type == 'DA-ZoeDepth':
                self.branch = target
                self._build_tree(branch_layout(cfg, target + '_branch.'))
                self.resizer = Resize(self.patch_process_shape[1], self.patch_process_shape[0], ensure_multiple_of=14)
        self._runtime_init()
        self._hook_invalidate()
        if self.branch is not None:
            self._init_constant_buffers(_get(self._branch_cfg(), 'n_bins', 64))

    def _branch_cfg(self):
        return self.coarse_branch_cfg if self.branch == 'coarse' else self.fine_branch_cfg

    # ------------------------------------------------------------------ reference API surface
    def load_dict(self, dict):
        """BP:121-127: unprefixed branch keys, strict."""
        if self.branch is None:
            raise NotImplementedError('Not support loading coarse and fine together')
        return getattr(self, self.branch + '_branch').load_state_dict(dict, strict=True)

    def get_save_dict(self):
        """BP:129-137: the unprefixed branch state dict (what PatchFusion(load_branch=True) reads back)."""
        if self.branch is None:
            raise NotImplementedError('Not support training coarse and fine together')
        return dict(getattr(self, self.branch + '_branch').state_dict())

    def init_synthetic_weights(self, seed=0):
        """Seeded random weights: the `<branch>_branch.*` subset of the PatchFusion synthetic weights of the same
        seed and branch config, so a single-branch model and a PatchFusion share their branch weights."""
        if self.branch is None:
            raise NotImplementedError('no branch is built for target %r' % (self.target,))
        cfg = {'coarse_branch': self.coarse_branch_cfg, 'fine_branch': self.fine_branch_cfg}
        self.load_state_dict(synthetic_state_dict(cfg, seed=seed, prefix=self.branch + '_branch.'), strict=True)
        return self

    # ------------------------------------------------------------------ engine plumbing
    def engine(self, shape=None):
        """The packed branch at processing size `shape` (default patch_process_shape).  A call at another size
        re-packs: the pos-embed resample depends on it."""
        from .engine import Engine
        if self.branch is None:
            raise NotImplementedError('no branch is built for target %r' % (self.target,))
        P = tuple(self.patch_process_shape if shape is None else shape)
        if self._engine is not None and self._engine.P != P:
            self.invalidate()
        if self._engine is None:
            p = next(self.parameters())
            if not p.is_cuda:
                raise RuntimeError('BaselinePretrain (H100): the hot path runs on libpf_b200 only; move the model to a '
                                   'CUDA device (there is no CPU fallback)')
            cfg = {'patch_process_shape': P, self.branch + '_branch': self._branch_cfg()}
            self._engine = Engine(cfg, self.state_dict(), p.device, parts=(self.branch,))
        return self._engine

    # ------------------------------------------------------------------ coarse target
    def _coarse_infer(self, image_lr):
        """One branch forward of the whole batch at image_lr's own size (BP:366), one graph per (B, h, w)."""
        B, _, h, w = image_lr.shape
        # dinov2 patch_embed.py:73-74
        assert h % 14 == 0, 'Input image height %d is not a multiple of patch height 14' % h
        assert w % 14 == 0, 'Input image width %d is not a multiple of patch width 14' % w
        eng = self.engine((h, w))
        x = eng.buf('in.image_lr', (B, 3, h, w), torch.float32)
        x.copy_(image_lr)
        out = eng.buf('out.depth', (B, h, w), torch.float32)

        def run():
            d, _ = eng.branch('coarse', x)
            out.copy_(d)
        self._graphed(('coarse', B, h, w), run)
        return out[:, None].clone()

    # ------------------------------------------------------------------ fine target
    def _tile_stage(self, eng, img, geom, sizes, io_raw, blk):
        """crop+resize -> fine branch per micro-batch; the depth (in the reused tile arena) is copied into its rows
        of the prediction block."""
        from . import ops
        H, W, h, w, ph, pw = geom
        s0 = 0
        for T in sizes:
            crops = eng.buf('tile.crops', (T, 3, ph, pw), torch.float32)
            ops.call('pf_crop_resize', img, H, W, io_raw[s0:s0 + T], T, h, w, ph, pw, crops, ops.stream_ptr())
            arena = eng.arena('tile', eng.branch_bytes('fine', T))
            fd, _ = eng.branch('fine', crops, ws=(arena, 0))
            blk[s0:s0 + T].copy_(fd)
            s0 += T

    def _compute_phase(self, eng, phase, img, geom, raw, process_num, shard):
        """Fine-branch predictions of this rank's tiles of the ordered tile list `raw` -> its block
        [block_rows, ph, pw] fp32 (round-robin: row j = tile rank + j * world)."""
        from .parallel import shard_indices, block_rows
        H, W, h, w, ph, pw = geom
        rank, world = (0, 1) if shard is None else shard
        n = len(raw)
        own = shard_indices(n, rank, world)
        blk = eng.buf('pred.blk.' + phase, (block_rows(n, world), ph, pw), torch.float32)
        if not own:
            return blk
        io_raw = eng.buf('io.raw.' + phase, (len(own), 2), torch.int32)
        io_raw.copy_(torch.tensor([raw[i] for i in own], dtype=torch.int32))
        sizes = self._micro_sizes(len(own), process_num)
        key = ('tiles', phase, tuple(sizes), blk.shape[0]) + tuple(geom)
        self._graphed(key, lambda: self._tile_stage(eng, img, geom, sizes, io_raw, blk))
        return blk

    @torch.no_grad()
    def forward(self, mode, image_lr, image_hr, depth_gt=None, crop_depths=None, crops_image_hr=None, bboxs=None,
                tile_cfg=None, cai_mode='m1', process_num=4, shard=None, group=None):
        """BP:333-419 (mode='infer').  depth_gt defaults to None so `Tester.run` can drive this model.
        Fine target only: `shard=(rank, world)` / `('emulate', W)` shards the tile list round-robin with one
        all-gather before the deterministic stitch (as `PatchFusion.forward`)."""
        if mode == 'train':
            raise NotImplementedError('training is out of scope of the H100 hot-path build (SURVEY.md §2 rows 10,12)')
        if self.target == 'coarse':
            depth = self._coarse_infer(image_lr)
            return depth, {'rgb': image_lr, 'depth_pred': depth, 'depth_gt': depth_gt}
        if self.target != 'fine':
            raise NotImplementedError
        if tile_cfg is None:
            tile_cfg = self.tile_cfg
        else:
            tile_cfg = self.prepare_tile_cfg(tile_cfg['image_raw_shape'], tile_cfg['patch_split_num'])
        assert image_hr.shape[0] == 1
        self._check_shard(shard, group)
        eng = self.engine()

        def compute(phase, img, geom, tiles, sh, plan):
            return self._compute_phase(eng, phase, img, geom, tiles, process_num, sh)

        n_calls = int(cai_mode[1:]) if cai_mode[0] == 'r' else 0      # BP:407-410: N calls, not N // process_num
        depth = self._tiled_forward(eng, image_hr, tile_cfg, cai_mode, process_num, shard, group, n_calls, compute)
        return depth, {}
