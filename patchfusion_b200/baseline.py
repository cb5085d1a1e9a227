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

Calibrated FP8 (an extension; the reference has no such keys): `branch_vit_precision` / `branch_dpt_precision` ('bf16'
default, or 'fp8_static') run the branch's DINOv2 qkv / fc1 / fc2 linears and its 19 covered DPT convs on E4M3 operands,
as PatchFusion's `vit_precision` / `dpt_precision` do for its branches.  Their tables `branch_vit_fp8_amax` /
`branch_dpt_fp8_amax` use PatchFusion's names for this branch ('<target>.<i>.<qkv|fc1|fc2>', '<target>.<conv>'), so
the `fine.*` entries of a PatchFusion table are a fine baseline's table and the other way round;
`BaselinePretrain.calibrate_fp8` fills them.  The tables are configuration: the state dict does not change.
PatchFusion's own keys (fusion_precision, vit_precision, dpt_precision and their tables) are accepted and ignored.
"""
import math
import os

import torch
import torch.nn as nn

from .model import AttrDict, Resize, TiledModel
from .params import _get, branch_layout, dpt_fp8_amax, dpt_fp8_layers, dpt_precision, synthetic_state_dict, \
    vit_fp8_amax, vit_fp8_layers, vit_precision


FP8_KEYS = ('branch_vit_precision', 'branch_vit_fp8_amax', 'branch_dpt_precision', 'branch_dpt_fp8_amax')


def save_baseline(model, cfg, out_dir, name):
    """Write `model` as the pair `tools/test.py DIR/<name>.py --ckp-path DIR/<name>.pth` evaluates: the config file of
    `cfg` (a load_config dict) whose model dict carries the model's FP8 keys, and {'model_state_dict':
    get_save_dict()}, the checkpoint format the reference's BaselinePretrain reads.  Returns the two paths."""
    from .config import save_config
    os.makedirs(out_dir, exist_ok=True)
    cfg = dict(cfg)
    cfg['model'] = dict(cfg['model'], **{k: getattr(model, k) for k in FP8_KEYS})
    paths = os.path.join(out_dir, name + '.py'), os.path.join(out_dir, name + '.pth')
    save_config(cfg, paths[0])
    torch.save({'model_state_dict': {k: v.detach().cpu() for k, v in model.get_save_dict().items()}}, paths[1])
    return paths


def _attr(cfg):
    if not isinstance(cfg, dict) and hasattr(cfg, 'to_dict'):
        cfg = cfg.to_dict()
    return AttrDict(dict(cfg))


class BaselinePretrain(TiledModel):
    def __init__(self, coarse_branch, fine_branch, sigloss, min_depth, max_depth, image_raw_shape=(2160, 3840),
                 patch_process_shape=(384, 512), patch_split_num=(4, 4), target='coarse', coarse_branch_zoe=None,
                 fusion_precision=None, fusion_fp8_amax=None, vit_precision=None, vit_fp8_amax=None,
                 dpt_precision=None, dpt_fp8_amax=None, branch_vit_precision='bf16', branch_vit_fp8_amax=None,
                 branch_dpt_precision='bf16', branch_dpt_fp8_amax=None):
        nn.Module.__init__(self)
        # fusion_precision selects the compute type of PatchFusion's Guided-Fusion U-Net and fusion_fp8_amax holds its
        # calibrated FP8 input scales; this model has no fusion stage, so a config that carries the keys (any value)
        # builds and packs exactly as without them.  vit_precision / vit_fp8_amax and dpt_precision / dpt_fp8_amax
        # (PatchFusion's FP8 ViT encoders and DPT decoders) are ignored the same way, so a PatchFusion config's values
        # never change a baseline: this model's FP8 switches are the branch_* keys.
        del fusion_precision, fusion_fp8_amax, vit_precision, vit_fp8_amax, dpt_precision, dpt_fp8_amax
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
        self.branch_vit_precision = branch_vit_precision
        self.branch_vit_fp8_amax = branch_vit_fp8_amax
        self.branch_dpt_precision = branch_dpt_precision
        self.branch_dpt_fp8_amax = branch_dpt_fp8_amax
        self._fp8_cfg()                     # ValueError on an unknown precision or a malformed table
        self._runtime_init()
        self._hook_invalidate()
        if self.branch is not None:
            self._init_constant_buffers(_get(self._branch_cfg(), 'n_bins', 64))

    def _fp8_cfg(self):
        """The validated FP8 keys as the engine config of this branch (PatchFusion's key names, this branch's table
        names): {} for the bf16 default, so the default engine is the one built without the keys."""
        keys = {k: getattr(self, k) for k in FP8_KEYS}
        keys.update(coarse_branch=self.coarse_branch_cfg, fine_branch=self.fine_branch_cfg)
        own = (self.branch,) if self.branch is not None else ()
        out = {}
        if vit_precision(keys, 'branch_vit_precision') == 'fp8_static':
            out.update(vit_precision='fp8_static', vit_fp8_amax=vit_fp8_amax(keys, 'branch_vit_fp8_amax', own))
        else:
            vit_fp8_amax(keys, 'branch_vit_fp8_amax', own)
        if dpt_precision(keys, 'branch_dpt_precision') == 'fp8_static':
            out.update(dpt_precision='fp8_static', dpt_fp8_amax=dpt_fp8_amax(keys, 'branch_dpt_fp8_amax', own))
        else:
            dpt_fp8_amax(keys, 'branch_dpt_fp8_amax', own)
        return out

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
        re-packs: the pos-embed resample depends on it.  The FP8 tables are read from the model's keys on every call: a
        changed table re-points the stage and drops the graphs captured with the old scales."""
        from .engine import Engine
        if self.branch is None:
            raise NotImplementedError('no branch is built for target %r' % (self.target,))
        P = tuple(self.patch_process_shape if shape is None else shape)
        fp8 = self._fp8_cfg()
        eng = self._engine
        if eng is not None and (eng.P != P or (eng.vit_fp8_static, eng.dpt_fp8_static) !=
                                ('vit_precision' in fp8, 'dpt_precision' in fp8)):
            self.invalidate()
        if self._engine is None:
            p = next(self.parameters())
            if not p.is_cuda:
                raise RuntimeError('BaselinePretrain (H100): the hot path runs on libpf_b200 only; move the model to a '
                                   'CUDA device (there is no CPU fallback)')
            cfg = dict(fp8, patch_process_shape=P, **{self.branch + '_branch': self._branch_cfg()})
            self._engine = Engine(cfg, self.state_dict(), p.device, parts=(self.branch,))
        else:
            if eng.vit_fp8_static and fp8['vit_fp8_amax'] != eng.vit_amax:
                eng.set_vit_fp8_amax(fp8['vit_fp8_amax'])
                self._graphs = {}
            if eng.dpt_fp8_static and fp8['dpt_fp8_amax'] != eng.dpt_amax:
                eng.set_dpt_fp8_amax(fp8['dpt_fp8_amax'])
                self._graphs = {}
        return self._engine

    def _check_tables(self, eng):
        """an 'fp8_static' branch without its calibration table refuses to run (calibration runs it in bf16)"""
        if eng.calib is not None:
            return
        for on, table, key in ((eng.vit_fp8_static, eng.vit_amax, 'vit'), (eng.dpt_fp8_static, eng.dpt_amax, 'dpt')):
            if on and table is None:
                raise RuntimeError("branch_%s_precision 'fp8_static' needs the calibrated input scales `branch_%s_fp8_amax`: "
                                   "run BaselinePretrain.calibrate_fp8 (or tools/calibrate_fp8.py) first" % (key, key))

    @torch.no_grad()
    def calibrate_fp8(self, image_lr, image_hr, cai_mode='m1', process_num=4, tile_cfg=None, reset=False):
        """Post-training calibration of the 'fp8_static' branch: runs forward(mode='infer') on the given images (the
        same arguments; the coarse target reads image_lr, one batch at its own size, the fine target the tiles of
        image_hr, batches, mixed geometry and rN modes drawing from `random` included) with the branch in bf16 on this
        model's panels, and takes, for each E4M3 ViT linear and each E4M3 DPT conv, the maximum over all images and
        tiles of its input's amax.  Each switched-on table is merged by max into `branch_vit_fp8_amax` /
        `branch_dpt_fp8_amax` (reset=True starts from empty tables).  Returns the ViT table, else the DPT table.  Runs
        eagerly: no graph of it is kept, and the graphs of earlier forwards are dropped."""
        fp8 = self._fp8_cfg()
        vit, dpt = 'vit_precision' in fp8, 'dpt_precision' in fp8
        if not vit and not dpt:
            raise ValueError("calibrate_fp8 needs branch_vit_precision or branch_dpt_precision 'fp8_static' (this "
                             "model: %r, %r)" % (self.branch_vit_precision, self.branch_dpt_precision))
        # the coarse target runs at image_lr's size: pack there first, so the forward keeps this engine
        eng = self.engine(tuple(image_lr.shape[-2:]) if self.target == 'coarse' and torch.is_tensor(image_lr) else None)
        eng.calib = {}
        graphs, self.use_cuda_graphs = self.use_cuda_graphs, False
        try:
            self.forward('infer', image_lr, image_hr, tile_cfg=tile_cfg, cai_mode=cai_mode, process_num=process_num)
            found = {k: v.item() for k, v in eng.calib.items()}
        finally:
            eng.calib = None
            self.use_cuda_graphs = graphs
            self._graphs = {}
        cfg = {'coarse_branch': self.coarse_branch_cfg, 'fine_branch': self.fine_branch_cfg}
        own = (self.branch,)
        for on, key, names, check in ((vit, 'branch_vit_fp8_amax', vit_fp8_layers(cfg, own), vit_fp8_amax),
                                      (dpt, 'branch_dpt_fp8_amax', dpt_fp8_layers(cfg, own), dpt_fp8_amax)):
            if not on:
                continue
            missing = [k for k in names if k not in found]
            if missing:
                raise RuntimeError('calibrate_fp8: no input amax for %s' % missing)
            table = {} if reset else dict(getattr(self, key) or {})
            for k in names:
                table[k] = max(table.get(k, 0.0), found[k]) if not math.isnan(found[k]) else found[k]
            setattr(self, key, check(dict(cfg, **{key: table}), key, own))      # ValueError on NaN / inf
        self.engine(eng.P)
        return dict(self.branch_vit_fp8_amax if vit else self.branch_dpt_fp8_amax)

    # ------------------------------------------------------------------ coarse target
    def _coarse_infer(self, image_lr):
        """One branch forward of the whole batch at image_lr's own size (BP:366), one graph per (B, h, w)."""
        B, _, h, w = image_lr.shape
        # dinov2 patch_embed.py:73-74
        assert h % 14 == 0, 'Input image height %d is not a multiple of patch height 14' % h
        assert w % 14 == 0, 'Input image width %d is not a multiple of patch width 14' % w
        eng = self.engine((h, w))
        self._check_tables(eng)
        x = eng.buf('in.image_lr', (B, 3, h, w), torch.float32)
        x.copy_(image_lr)
        out = eng.buf('out.depth', (B, h, w), torch.float32)

        def run():
            d, _ = eng.branch('coarse', x)
            out.copy_(d)
        self._graphed(('coarse', B, h, w), run)
        return out[:, None].clone()

    # ------------------------------------------------------------------ fine target
    def _tile_stage(self, eng, img, geom, sizes, io_raw, io_img, blk):
        """crop+resize -> fine branch per micro-batch (a micro-batch may mix images: io_img gives each tile's, None =
        image 0); the depth (in the reused tile arena) is copied into its rows of the prediction block."""
        ph, pw = self.patch_process_shape
        s0 = 0
        for T in sizes:
            crops = eng.buf('tile.crops', (T, 3, ph, pw), torch.float32)
            self._crop(img, geom, io_raw[s0:s0 + T], None if io_img is None else io_img[s0:s0 + T], crops)
            arena = eng.arena('tile', eng.branch_bytes('fine', T))
            fd, _ = eng.branch('fine', crops, ws=(arena, 0))
            blk[s0:s0 + T].copy_(fd)
            s0 += T

    def _compute_phase(self, eng, phase, img, geom, raw, process_num, shard):
        """Fine-branch predictions of this rank's tiles of the ordered tile list `raw` ((image, y, x) items of img
        [B,3,H,W], or (y, x) tiles of image 0) -> its block [block_rows, ph, pw] fp32 (round-robin: row j = tile
        rank + j * world).  geom: one (H, W, h, w, ph, pw), or one per image of a mixed batch (img is then its crop
        table)."""
        from .parallel import shard_indices, block_rows
        ph, pw = self.patch_process_shape
        mixed = self.is_mixed(geom)
        rank, world = (0, 1) if shard is None else shard
        n = len(raw)
        own = shard_indices(n, rank, world)
        blk = eng.buf('pred.blk.' + phase, (block_rows(n, world), ph, pw), torch.float32)
        if not own:
            return blk
        chunk, images = self.split_tiles([raw[i] for i in own])
        io_raw = eng.buf('io.raw.' + phase, (len(own), 2), torch.int32)
        io_raw.copy_(torch.tensor(chunk, dtype=torch.int32))
        B = len(geom) if mixed else img.shape[0] if img.dim() == 4 else 1
        io_img = None
        if B > 1 or mixed:
            io_img = eng.buf('io.img.' + phase, (len(own),), torch.int32)
            io_img.copy_(torch.tensor(images, dtype=torch.int32))
        sizes = self._micro_sizes(len(own), process_num)
        key = ('tiles', phase, tuple(sizes), blk.shape[0], B) + tuple(geom)
        self._graphed(key, lambda: self._tile_stage(eng, img, geom, sizes, io_raw, io_img, blk))
        return blk

    @torch.no_grad()
    def forward(self, mode, image_lr, image_hr, depth_gt=None, crop_depths=None, crops_image_hr=None, bboxs=None,
                tile_cfg=None, cai_mode='m1', process_num=4, shard=None, group=None):
        """BP:333-419 (mode='infer').  depth_gt defaults to None so `Tester.run` can drive this model.
        Fine target: image_hr [B,3,H,W] with any B >= 1 (extension: the reference takes B = 1) -> [B,1,H',W']; the
        tiles of all images are micro-batched together and image b equals the single-image call made after images
        0..b-1 from the same `random` state.  `shard=(rank, world)` / `('emulate', W)` shards the tile list
        round-robin with one all-gather before the deterministic stitch (as `PatchFusion.forward`).  The fine target
        also takes a mixed batch (lists of images, tile_cfgs and modes) and then returns a list, as
        `PatchFusion.forward`; the coarse target takes one image_lr batch of one size."""
        if mode == 'train':
            raise NotImplementedError('training is out of scope of the H100 hot-path build (SURVEY.md §2 rows 10,12)')
        if self.target == 'coarse':
            if isinstance(image_lr, (list, tuple)):
                raise ValueError('the coarse target takes image_lr as one [B, 3, h, w] tensor, not a list')
            depth = self._coarse_infer(image_lr)
            return depth, {'rgb': image_lr, 'depth_pred': depth, 'depth_gt': depth_gt}
        if self.target != 'fine':
            raise NotImplementedError
        image_hr, tile_cfg, cai_mode, as_list = self._batch_inputs(image_hr, tile_cfg, cai_mode)
        assert len(image_hr) >= 1
        self._check_shard(shard, group)
        eng = self.engine()
        self._check_tables(eng)

        def compute(phase, img, geom, tiles, sh, plan):
            return self._compute_phase(eng, phase, img, geom, tiles, process_num, sh)

        n_calls = lambda m: int(m[1:])              # BP:407-410: N calls, not N // process_num
        depth = self._tiled_forward(eng, image_hr, tile_cfg, cai_mode, process_num, shard, group, n_calls, compute)
        if as_list and not isinstance(depth, list):
            depth = list(depth.split(1))
        return depth, {}
