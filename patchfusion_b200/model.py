"""Drop-in `PatchFusion` for the reference's `estimator.models.patchfusion.PatchFusion` (inference path).

Same constructor dict / `from_pretrained()` / `state_dict()` key layout / `forward(mode='infer', image_lr,
image_hr, tile_cfg, cai_mode, process_num)` contract and error behaviour as reference
`estimator/models/patchfusion.py:55-453` + `estimator/models/baseline_pretrain.py:91-331`; the arithmetic runs on
libpf_b200 (sm_90a) through `Engine`.  There is no CPU path: calling forward on CPU tensors raises.
"""
import math
import os
import random

import numpy as np
import torch
import torch.nn as nn

from .params import ParamTree, _get, state_layout, synthetic_state_dict, relative_position_index

try:
    from huggingface_hub import PyTorchModelHubMixin
except Exception:                                   # pragma: no cover
    class PyTorchModelHubMixin:                     # minimal stand-in when huggingface_hub is absent
        pass


class AttrDict(dict):
    """Attribute-style view of nested config dicts (the reference reads `config.coarse_branch.type`)."""

    def __init__(self, d=None):
        super().__init__()
        for k, v in (d or {}).items():
            self[k] = AttrDict(v) if isinstance(v, dict) else v

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)

    def __setattr__(self, k, v):
        self[k] = v

    def to_dict(self):
        return {k: (v.to_dict() if isinstance(v, AttrDict) else v) for k, v in self.items()}

    def to_json_file(self, path):                   # `tools/convert_huggingface.py:79`
        import json
        with open(path, 'w') as f:
            json.dump(self.to_dict(), f, indent=2)


class Resize:
    """`model.resizer`: bilinear align_corners=True to patch_process_shape (depth_anything/transform.py:127-129 with
    keep_aspect_ratio=False => always exactly (h, w), as used at patchfusion.py:94).

    ensure_multiple_of > 1 (BaselinePretrain, baseline_pretrain.py:75,85): each side is rounded to the nearest
    multiple, computed from the input size exactly as transform.py:56-57 / 111-113 do ('minimal', no aspect ratio
    kept): (384, 512) -> 378 x 518, (392, 518) unchanged."""

    def __init__(self, width, height, ensure_multiple_of=1):
        self.w, self.h = width, height
        self.multiple = ensure_multiple_of

    def out_size(self, height, width):
        """(h, w) of the resized image for an input of height x width."""
        if self.multiple == 1:
            return int(self.h), int(self.w)
        m = self.multiple
        h = int(np.round(self.h / height * height / m) * m)
        w = int(np.round(self.w / width * width / m) * m)
        return h, w

    def __call__(self, x):
        return nn.functional.interpolate(x, self.out_size(*x.shape[-2:]), mode='bilinear', align_corners=True)


def _gauss_kernel(ksize, sigma):
    i = np.arange(ksize, dtype=np.float64) - (ksize - 1) / 2
    k = np.exp(-(i * i) / (2.0 * sigma * sigma))
    return (k / k.sum()).astype(np.float32)


def generatemask(size):
    """Gaussian blend mask of `estimator/models/utils.py:38-47` without OpenCV: 1 inside the central 80 %, separable
    Gaussian blur (k = 2*ceil(2*sigma)+1, sigma = int(H/16), BORDER_REFLECT_101), min-max normalised."""
    H, W = int(size[0]), int(size[1])
    mask = np.zeros((H, W), dtype=np.float32)
    sigma = int(H / 16)
    k = int(2 * np.ceil(2 * int(H / 16)) + 1)
    mask[int(0.1 * H):H - int(0.1 * H), int(0.1 * W):W - int(0.1 * W)] = 1
    ker = _gauss_kernel(k, float(sigma))
    r = k // 2

    def blur_rows(a):       # convolve along axis 1
        p = np.pad(a, ((0, 0), (r, r)), mode='reflect')
        cs = np.zeros_like(a, dtype=np.float32)
        for j in range(k):
            cs += ker[j] * p[:, j:j + a.shape[1]]
        return cs

    m = blur_rows(mask)
    m = blur_rows(m.T.copy()).T
    m = (m - m.min()) / (m.max() - m.min())
    return np.ascontiguousarray(m, dtype=np.float32)


class TiledModel(ParamTree):
    """What `PatchFusion` and `BaselinePretrain` share, as the reference's `PatchFusion(BaselinePretrain)` does: tile
    configuration, `make_lr`, blend masks, CUDA-graph replay, and the tiled forward of one image (regular passes
    flattened into one ordered tile list, the random phase, the deterministic stitch and the tile sharding).  The
    subclass supplies `compute(phase, img, geom, tiles, shard, plan)`: this rank's prediction block of the tile list."""

    # pf_stitch_gather takes at most 4096 tiles per call: the random phase is computed and stitched in chunks of at
    # most this many tiles, each continuing from the previous sums, so the canvas equals one pass bit for bit
    random_chunk = 4096

    def _runtime_init(self):
        self._engine = None
        self._graphs = {}
        self.graph_launches = 0
        self.use_cuda_graphs = os.environ.get('PF_B200_GRAPHS', '1') != '0'
        self.partition = os.environ.get('PF_B200_PARTITION', 'greedy')
        self._mask_cache = {}

    def _hook_invalidate(self):
        # sub-module loads (model.fine_branch.load_state_dict(sd), as the load_branch constructor path does) and
        # .to()/.half() on a sub-module must drop the packed bf16 panels too: hook every container node
        for m in self.modules():
            if m is not self:
                m.register_load_state_dict_post_hook(lambda mod, inc, _s=self: _s.invalidate())

    def _init_constant_buffers(self, n_bins):
        """constant buffers exactly as the reference constructs them"""
        with torch.no_grad():
            for name, buf in self.named_buffers():
                if name.endswith('relative_position_index'):
                    buf.copy_(relative_position_index())
                elif name.endswith('k_idx'):
                    buf.copy_(torch.arange(buf.numel()).view(buf.shape))
                elif name.endswith('K_minus_1'):
                    buf.fill_(float(n_bins - 1))
                elif name.endswith('running_var'):
                    buf.fill_(1.0)

    # ------------------------------------------------------------------ reference API surface
    def prepare_tile_cfg(self, image_raw_shape, patch_split_num):
        assert image_raw_shape[0] % (2 * patch_split_num[0]) == 0, \
            'image height should be divisible by 2 * patch_split_num[0]'
        assert image_raw_shape[1] % (2 * patch_split_num[1]) == 0, \
            'image width should be divisible by 2 * patch_split_num[1]'
        pps = self.patch_process_shape
        patch_reensemble_shape = (pps[0] * patch_split_num[0], pps[1] * patch_split_num[1])
        patch_raw_shape = (image_raw_shape[0] // patch_split_num[0], image_raw_shape[1] // patch_split_num[1])
        return {'patch_split_num': patch_split_num, 'patch_reensemble_shape': patch_reensemble_shape,
                'patch_raw_shape': patch_raw_shape, 'image_raw_shape': image_raw_shape,
                'raw_h_split_point': [int(patch_raw_shape[0] * i) for i in range(patch_split_num[0])],
                'raw_w_split_point': [int(patch_raw_shape[1] * i) for i in range(patch_split_num[1])]}

    def load_state_dict(self, *a, **kw):
        self.invalidate()
        return super().load_state_dict(*a, **kw)

    def _apply(self, fn, *a, **kw):
        self.invalidate()
        return super()._apply(fn, *a, **kw)

    @torch.no_grad()
    def make_lr(self, image_hr):
        """`image_lr = model.resizer(image)` of `tools/test_single_forward.py:13-14` on the device (same bilinear
        align_corners=True resample, pf_crop_resize with one whole-image tile)."""
        from . import ops
        img = image_hr[0].float().contiguous()
        H, W = img.shape[-2:]
        ph, pw = self.resizer.out_size(H, W)
        out = torch.empty((1, 3, ph, pw), dtype=torch.float32, device=img.device)
        org = torch.zeros((1, 2), dtype=torch.int32, device=img.device)
        ops.call('pf_crop_resize', img, H, W, org, 1, H, W, ph, pw, out, ops.stream_ptr())
        return out

    def _mask(self, size, device):
        key = (tuple(size), str(device))
        if key not in self._mask_cache:
            self._mask_cache[key] = torch.tensor(generatemask(size) + 1e-3, device=device).contiguous()
        return self._mask_cache[key]

    # ------------------------------------------------------------------ tiling
    def _graphed(self, key, fn):
        """Run `fn` (a fixed kernel sequence over static buffers) through a CUDA graph: first call runs eagerly
        (allocating the engine buffers and caching the TMA maps) and captures, later calls replay.  One graph per
        (phase, micro-batch sizes, geometry): the ~2800 launches of a 4K P49 image collapse into one host call."""
        from . import lib
        if not self.use_cuda_graphs or lib.PROFILER is not None:
            return fn()
        ent = self._graphs.get(key)
        eng = self._engine
        if ent is None or ent[2] != eng.generation:     # workspaces were (re)allocated: old graphs point at freed memory
            fn()
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            n0 = lib.launch_count()
            with torch.cuda.graph(g):
                fn()
            self._graphs[key] = (g, lib.launch_count() - n0, eng.generation)
            return None
        ent[0].replay()
        self.graph_launches += ent[1]          # kernels executed by the replay (for bench.py's gpu_launches)
        return None

    def invalidate(self):
        """Drop the packed-weight engine and the captured graphs (call after editing parameters in place; state-dict
        loads and `.to()` on the model or any sub-module do it automatically)."""
        self._engine, self._graphs = None, {}

    def _micro_sizes(self, n, process_num):
        nchunk = -(-n // process_num)
        if self.partition == 'balanced':        # e.g. 49 tiles, process_num 9 -> 9,8,8,8,8,8
            return [n // nchunk + (1 if i < n % nchunk else 0) for i in range(nchunk)]
        return [min(process_num, n - i * process_num) for i in range(nchunk)]     # the reference's split (BP:293)

    @staticmethod
    def _chunks(n, size):
        """[start, stop) ranges of the random phase's chunks: n tiles in order, at most `size` per chunk."""
        return [(s, min(s + size, n)) for s in range(0, n, size)]

    @staticmethod
    def _check_shard(shard, group):
        if shard is not None and shard[0] != 'emulate':
            import torch.distributed as dist
            assert dist.is_initialized() and dist.get_world_size(group) == shard[1] and dist.get_rank(group) == shard[0], \
                'shard=(rank, world) must match the process group the blocks are gathered over'

    def _exchange(self, compute, shard, group):
        """The ONE collective of the tile-sharded path: all-gather of the per-rank prediction blocks.
        shard=None: single device.  shard=('emulate', W): the W ranks are computed one after the other in this
        process (test hook for 1-GPU boxes; same blocks, same stitch)."""
        self._real_shard = shard is not None and shard[0] != 'emulate'
        if shard is None:
            return compute(None)
        if shard[0] == 'emulate':
            return torch.cat([compute((r, shard[1])).clone() for r in range(shard[1])])
        from .parallel import gather_blocks
        return gather_blocks(compute(shard), shard[1], group)

    def _stitch_phase(self, eng, phase, full, origins, world, th, tw, mask, up, base, canvas, want, plan=None):
        """pf_stitch_gather over the global tile list (deterministic order) -> requested canvases."""
        from . import ops
        from .parallel import slot_table
        CH, CW = canvas
        n = len(origins)
        slots = slot_table(n, world, plan)
        tab = eng.buf('stitch.tab.' + phase, (n, 3), torch.int32)
        tab.copy_(torch.tensor([(oy, ox, sl) for (oy, ox), sl in zip(origins, slots)], dtype=torch.int32))
        dev = full.device
        outs = {k: torch.empty((CH, CW), dtype=torch.float32, device=dev) for k in want}
        ops.call('pf_stitch_gather', full, tab, n, th, tw, mask, up[0], up[1],
                 base[0] if base else None, base[1] if base else None, CH, CW,
                 outs.get('num'), outs.get('den'), outs.get('avg'), ops.stream_ptr())
        return outs

    def _draw_random_boxes(self, n_calls, process_num, H, W, h, w, shard, group, dev):
        """Random tile origins in the reference's draw order (baseline_pretrain.py:155-156: process_num rows, then ONE
        shared column per call).  Under real sharding rank 0's draws are broadcast so every rank stitches the same
        list (all ranks still advance their own `random` state identically)."""
        boxes = []
        for _ in range(n_calls):
            ys = [random.randint(0, H - h - 1) for _ in range(process_num)]
            x0 = random.randint(0, W - w - 1)
            boxes += [(y, x0) for y in ys]
        if shard is not None and shard[0] != 'emulate' and boxes:
            import torch.distributed as dist
            t = torch.tensor(boxes, dtype=torch.int32, device=dev if dist.get_backend(group) == 'nccl' else 'cpu')
            dist.broadcast(t, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
            boxes = [tuple(b) for b in t.cpu().tolist()]
        return boxes

    def _tiled_forward(self, eng, image_hr, tile_cfg, cai_mode, process_num, shard, group, n_random_calls, compute,
                       image_lr=None, plan_fn=None):
        """Tiled inference of one image: the regular passes (baseline_pretrain.py:221-331, patchfusion.py:417-439) are
        independent tiles whose stitch is a weighted sum, so all passes are flattened into one ordered tile list and
        micro-batched; rN modes then resize the canvas to image_raw_shape and add `n_random_calls` calls of
        `process_num` random tiles.  image_lr (PatchFusion) goes into its static buffer; plan_fn(n) gives the rank of
        each regular tile (None: round-robin)."""
        from . import ops
        dev = image_hr.device
        H, W = tile_cfg['image_raw_shape']
        assert tuple(image_hr.shape[-2:]) == (H, W), 'image_hr must already be at image_raw_shape'
        h, w = tile_cfg['patch_raw_shape']
        ph, pw = self.patch_process_shape
        RH, RW = tile_cfg['patch_reensemble_shape']
        geom = (H, W, h, w, ph, pw)
        world = 1 if shard is None else shard[1]
        # inputs into static buffers (stable addresses for the captured graphs)
        img = eng.buf('in.image_hr', (3, H, W), torch.float32)
        img.copy_(image_hr[0])
        if image_lr is not None:
            eng.buf('in.image_lr', (1, 3, ph, pw), torch.float32).copy_(image_lr)
        mask = self._mask((ph, pw), dev)
        offsets = [((0, 0), (0, 0))]
        if cai_mode == 'm2' or cai_mode[0] == 'r':
            offsets += [((0, w // 2), (0, pw // 2)), ((h // 2, 0), (ph // 2, 0)), ((h // 2, w // 2), (ph // 2, pw // 2))]
        raw, proc = [], []
        for (oy, ox), (py, px) in offsets:
            assert ox >= 0 and oy >= 0
            ny, nx = (H - oy) // h, (W - ox) // w
            raw += [(h * a + oy, w * b + ox) for a in range(ny) for b in range(nx)]
            proc += [(ph * a + py, pw * b + px) for a in range(ny) for b in range(nx)]
        is_r = cai_mode[0] == 'r'
        plan = plan_fn(len(raw)) if plan_fn is not None else None
        full = self._exchange(lambda sh: compute('reg', img, geom, raw, sh, plan), shard, group)
        outs = self._stitch_phase(eng, 'reg', full, proc, world, ph, pw, mask, (0, 0), None, (RH, RW),
                                  ('num', 'den') if is_r else ('avg',), plan)
        if is_r:
            n2 = torch.empty((H, W), dtype=torch.float32, device=dev)
            d2 = torch.empty_like(n2)
            ops.call('pf_stitch_resize', outs['num'], outs['den'], RH, RW, H, W, n2, d2, ops.stream_ptr())
            boxes = self._draw_random_boxes(n_random_calls, process_num, H, W, h, w, shard, group, dev)
            if boxes:
                mask_r = self._mask((h, w), dev)
                base = (n2, d2)
                chunks = self._chunks(len(boxes), self.random_chunk)
                for s0, s1 in chunks:
                    part = boxes[s0:s1]
                    last = s1 == len(boxes)
                    full = self._exchange(lambda sh: compute('rnd', img, geom, part, sh, None), shard, group)
                    outs = self._stitch_phase(eng, 'rnd', full, part, world, ph, pw, mask_r, (h, w), base, (H, W),
                                              ('avg',) if last else ('num', 'den'))
                    if not last:
                        base = (outs['num'], outs['den'])
            else:
                outs = {'avg': n2 / d2}
        return outs['avg'][None, None]


class PatchFusion(TiledModel, PyTorchModelHubMixin):
    def __init__(self, config):
        nn.Module.__init__(self)
        if not isinstance(config, dict) and hasattr(config, 'to_dict'):
            config = config.to_dict()
        config = AttrDict(dict(config))
        # the HF-dict constructor branch of the reference (patchfusion.py:70-78)
        config.load_branch = bool(config.get('load_branch', False))
        self.config = config
        self.min_depth = config.min_depth
        self.max_depth = config.max_depth
        self.patch_process_shape = config.patch_process_shape
        self.tile_cfg = self.prepare_tile_cfg(config.image_raw_shape, config.patch_split_num)
        self.coarse_branch_cfg = config.coarse_branch
        for br in (config.coarse_branch, config.fine_branch):
            if br.type not in ('ZoeDepth', 'DA-ZoeDepth'):
                raise NotImplementedError
        self.resizer = Resize(config.patch_process_shape[1], config.patch_process_shape[0])
        self._build_tree(state_layout(config))      # raises ValueError / NotImplementedError like the reference
        self.consistency_training = False
        self._runtime_init()
        self._coarse = None
        # coarse branch + G2L (batch 1) on a side stream next to the first fine branch: measured in DESIGN.md
        self.overlap_coarse = os.environ.get('PF_B200_OVERLAP_COARSE', '1') != '0'
        self._side_stream = None
        # tile-sharded forward: 'owner' = rank 0 computes the per-image coarse branch + G2L, takes `owner_cost_tiles`
        # fewer tiles and broadcasts the packed result; 'replicate' = every rank computes it (no broadcast)
        self.shard_coarse = os.environ.get('PF_B200_SHARD_COARSE', 'owner')
        self.owner_cost_tiles = float(os.environ.get('PF_B200_OWNER_COST', '2.7'))
        self._pack = None
        self._hook_invalidate()
        if config.load_branch:
            for which, path in zip(('coarse_branch', 'fine_branch'), config.pretrain_model):
                sd = torch.load(path, map_location='cpu')['model_state_dict']
                getattr(self, which).load_state_dict(sd, strict=True)
        self._init_constant_buffers(_get(config.coarse_branch, 'n_bins', 64))

    # ------------------------------------------------------------------ reference API surface
    def load_dict(self, dict):
        return self.load_state_dict(dict, strict=False)

    def get_save_dict(self):
        return {k: v for k, v in self.state_dict().items() if 'coarse_branch' not in k and 'fine_branch' not in k}

    def init_synthetic_weights(self, seed=0):
        """Seeded random weights (no checkpoints are reachable offline)."""
        self.load_state_dict(synthetic_state_dict(self.config, seed=seed), strict=True)
        return self

    # ------------------------------------------------------------------ engine plumbing
    def engine(self, device=None):
        from .engine import Engine
        if self._engine is None:
            p = next(self.parameters())
            if not p.is_cuda:
                raise RuntimeError('PatchFusion (H100): the hot path runs on libpf_b200 only; move the model to a '
                                   'CUDA device (there is no CPU fallback)')
            self._engine = Engine(self.config, self.state_dict(), p.device)
        return self._engine

    def invalidate(self):
        super().invalidate()
        self._pack = None

    # ------------------------------------------------------------------ stage-level entry points (NCHW fp32 views)
    @staticmethod
    def _nchw(m):
        return m.t[..., :m.C].float().permute(0, 3, 1, 2).contiguous()

    @torch.no_grad()
    def coarse_forward(self, image_lr):
        d, feats = self.engine().branch('coarse', image_lr.float().contiguous())
        return d[:, None].clone(), [self._nchw(f) for f in feats]

    @torch.no_grad()
    def fine_forward(self, image_hr_crop):
        d, feats = self.engine().branch('fine', image_hr_crop.float().contiguous())
        return d[:, None].clone(), [self._nchw(f) for f in feats]

    def _to_map(self, x):
        """NCHW fp32 tensor -> engine Map (NHWC bf16, channels padded to 8)."""
        from .engine import Map
        from .ops import pad_to
        B, C, H, W = x.shape
        t = torch.zeros((B, H, W, pad_to(C, 8)), dtype=torch.bfloat16, device=x.device)
        t[..., :C] = x.permute(0, 2, 3, 1).to(torch.bfloat16)
        return Map(t, C)

    @torch.no_grad()
    def coarse_postprocess_test(self, coarse_prediction, coarse_features, bboxs, bboxs_feat):
        """`patchfusion.py:240-257`: ROI crop-zoom of the coarse depth and taps for the boxes `bboxs_feat` (T,5:
        batch index, x1, y1, x2, y2 in patch_process units).  NCHW fp32 in / out like the reference."""
        from . import ops
        boxes = bboxs_feat[:, 1:].float().contiguous()
        T = boxes.shape[0]
        P = self.patch_process_shape
        feats = []
        for f in coarse_features:
            m = self._to_map(f.float())
            h, w = m.hw
            out = torch.zeros((T, h, w, m.t.shape[-1]), dtype=torch.bfloat16, device=f.device)
            ops.roi_crop_zoom(m.t, m.C, boxes, h / P[0], out)
            feats.append(out[..., :m.C].float().permute(0, 3, 1, 2).contiguous())
        d = coarse_prediction.float().contiguous()
        droi = torch.zeros((T,) + tuple(d.shape[-2:]), dtype=torch.float32, device=d.device)
        ops.roi_crop_zoom(d[0, 0].contiguous(), 1, boxes, d.shape[-2] / P[0], droi)
        return {'coarse_depth_roi': droi[:, None], 'coarse_feats_roi': feats}

    @torch.no_grad()
    def infer_forward(self, imgs_crop, bbox_feat_forward, tile_temp, coarse_temp_dict=None):
        """`patchfusion.py:343-356`: fine branch + guided fusion of the given crops (T,3,h,w in [0,1]) against the
        whole-image coarse outputs in `tile_temp` ({'coarse_prediction', 'coarse_features'}, NCHW fp32).  As in the
        reference the G2L maps are recomputed from `tile_temp` on every call; `coarse_temp_dict` (the precomputed ROI
        crops) is accepted for signature compatibility - the kernels re-derive the crops from the boxes."""
        eng = self.engine()
        crops = imgs_crop.float().contiguous()
        boxes = bbox_feat_forward[:, 1:].float().contiguous()
        cf = [self._to_map(f.float()) for f in tile_temp['coarse_features']]
        cd = tile_temp['coarse_prediction'].float()[0, 0].contiguous()
        g2l = eng.g2l(cf)
        fd, ff = eng.branch('fine', crops)
        return eng.fusion(crops, boxes, fd, ff, cd, cf, g2l)[:, None].clone()

    # ------------------------------------------------------------------ tiling
    def _coarse_stage(self, eng, lr, pack=False):
        """coarse branch + G2L of the whole image.  pack=True (tile-sharded owner): the results are copied into the
        contiguous pack buffer that is broadcast, and every later stage reads the pack."""
        cd, cf = eng.branch('coarse', lr)
        res = (cd[0], cf, eng.g2l(cf))
        if not pack:
            self._coarse = res
            return
        dst = self._pack[1]
        dst[0].copy_(res[0])
        for d, m in zip(dst[1] + dst[2], res[1] + res[2]):
            d.t.copy_(m.t)
        self._coarse = dst

    def _ensure_pack(self, eng, lr):
        """Pack buffer for the coarse results (coarse depth fp32, 6 coarse maps, 6 G2L maps; 256-B aligned segments).
        Its layout follows from the model geometry alone; the first call runs the coarse stage once to read the
        shapes off the stage outputs (every rank, outside any timed region)."""
        if self._pack is not None and self._pack[2] is eng:
            self._coarse = self._pack[1]
            return self._pack[0]
        from .engine import Map
        cd, cf = eng.branch('coarse', lr)
        g2l = eng.g2l(cf)
        items = [(cd[0].shape, torch.float32, None)] + [(m.t.shape, m.t.dtype, m.C) for m in cf + g2l]
        offs, total = [], 0
        for shape, dt, _ in items:
            offs.append(total)
            total += (int(np.prod(shape)) * torch.empty((), dtype=dt).element_size() + 255) // 256 * 256
        buf = eng.buf('coarse.pack', (total,), torch.uint8)
        views = []
        for (shape, dt, C), o in zip(items, offs):
            nb = int(np.prod(shape)) * torch.empty((), dtype=dt).element_size()
            t = buf[o:o + nb].view(dt).view(tuple(shape))
            views.append(t if C is None else Map(t, C))
        self._pack = (buf, (views[0], views[1:1 + len(cf)], views[1 + len(cf):]), eng)
        self._coarse = self._pack[1]
        return buf

    def _fine_stage(self, eng, img, T, geom, raw):
        """crop+resize -> fine branch for the T tiles whose raw origins are the device rows `raw` ([T,2] int32)."""
        from . import ops
        H, W, h, w, ph, pw = geom
        crops = eng.buf('tile.crops', (T, 3, ph, pw), torch.float32)
        ops.call('pf_crop_resize', img, H, W, raw, T, h, w, ph, pw, crops, ops.stream_ptr())
        # ONE arena for the tile stages, sized for the largest micro-batch: [fine branch | fusion]
        nb = (eng.branch_bytes('fine', T) + 255) // 256 * 256
        arena = eng.arena('tile', nb + eng.fusion_bytes(T, self._coarse[2]))
        fd, ff = eng.branch('fine', crops, ws=(arena, 0))
        return crops, fd, ff, (arena, nb)

    def _fusion_stage(self, eng, fine, boxes, out):
        """guided fusion of one micro-batch; the fused depth goes straight into its rows `out` of the prediction block."""
        cd, cf, g2l = self._coarse
        crops, fd, ff, ws = fine
        eng.fusion(crops, boxes, fd, ff, cd, cf, g2l, depth_out=out, ws=ws)

    def _image_stage(self, eng, lr, img, geom, sizes, io_raw, io_box, blk, with_coarse, part='all'):
        """The static kernel sequence of one phase of one image on this rank: [coarse branch + G2L] and the
        micro-batches (fine branch + fusion each).  The coarse stage has no dependency on the first fine branch, so it
        runs on a side stream next to it (its batch-1 kernels fill a fraction of the SMs).
        part='pre' / 'post' (tile-sharded, non-owner ranks): the fine branch of the first micro-batch runs BEFORE the
        broadcast of the owner's coarse results arrives, everything else after it."""
        from . import lib
        if part == 'pre':
            self._pending_fine = self._fine_stage(eng, img, sizes[0], geom, io_raw[:sizes[0]])
            return
        if part == 'post':
            T0 = sizes[0]
            self._fusion_stage(eng, self._pending_fine, io_box[:T0], blk[:T0])
            io_raw, io_box, blk, sizes = io_raw[T0:], io_box[T0:], blk[T0:], sizes[1:]
        cur = torch.cuda.current_stream()
        side = None
        if with_coarse:
            if self.overlap_coarse and lib.PROFILER is None and sizes:
                if self._side_stream is None:
                    self._side_stream = torch.cuda.Stream()
                side = self._side_stream
                side.wait_stream(cur)
                with torch.cuda.stream(side):
                    self._coarse_stage(eng, lr)
            else:
                self._coarse_stage(eng, lr)
        s0 = 0
        for T in sizes:
            fine = self._fine_stage(eng, img, T, geom, io_raw[s0:s0 + T])
            if side is not None:
                cur.wait_stream(side)
                side = None
            self._fusion_stage(eng, fine, io_box[s0:s0 + T], blk[s0:s0 + T])
            s0 += T

    def _compute_phase(self, eng, phase, lr, img, geom, raw, process_num, shard, plan=None, group=None):
        """Fused predictions of this rank's tiles of the (global, ordered) tile list `raw` -> its block
        [block_rows, ph, pw] fp32 (row j = the j-th tile of the list that `plan` gives to this rank)."""
        from .parallel import shard_indices, block_rows
        H, W, h, w, ph, pw = geom
        rank, world = (0, 1) if shard is None else shard
        n = len(raw)
        own = shard_indices(n, rank, world, plan)
        blk = eng.buf('pred.blk.' + phase, (block_rows(n, world, plan), ph, pw), torch.float32)
        with_coarse = phase == 'reg'
        owner_mode = with_coarse and shard is not None and self.shard_coarse == 'owner'
        real = shard is not None and self._real_shard
        if owner_mode:
            # rank 0 computes coarse + G2L into the pack and broadcasts it; the others start on their fine branch
            pack = self._ensure_pack(eng, lr)
            if rank == 0:
                self._graphed(('coarse.pack',) + tuple(geom), lambda: self._coarse_stage(eng, lr, pack=True))
            with_coarse = False
        if not own:
            if owner_mode and real:
                self._broadcast_pack(pack, group)
            return blk
        io_raw = eng.buf('io.raw.' + phase, (len(own), 2), torch.int32)
        io_box = eng.buf('io.box.' + phase, (len(own), 4), torch.float32)
        fx, fy = np.float32(1 / W * pw), np.float32(1 / H * ph)
        chunk = [raw[i] for i in own]
        io_raw.copy_(torch.tensor(chunk, dtype=torch.int32))
        # boxes exactly as baseline_pretrain.py:268-282: int pixel box * fp32 factor
        io_box.copy_(torch.from_numpy(np.array(
            [[np.float32(x) * fx, np.float32(y) * fy, np.float32(x + w) * fx, np.float32(y + h) * fy]
             for (y, x) in chunk], dtype=np.float32)))
        sizes = self._micro_sizes(len(own), process_num)
        key = ('image', phase, tuple(sizes), blk.shape[0], with_coarse) + tuple(geom)
        run = lambda part: self._graphed(key + (part,), lambda: self._image_stage(
            eng, lr, img, geom, sizes, io_raw, io_box, blk, with_coarse, part))
        if owner_mode and real:
            if rank != 0:
                run('pre')
            self._broadcast_pack(pack, group)
            run('post' if rank != 0 else 'all')
        else:
            run('all')
        return blk

    @staticmethod
    def _broadcast_pack(pack, group):
        import torch.distributed as dist
        dist.broadcast(pack, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)

    @torch.no_grad()
    def forward(self, mode, image_lr, image_hr, depth_gt=None, crops_image_hr=None, crop_depths=None, bboxs=None,
                tile_cfg=None, cai_mode='m1', process_num=4, shard=None, group=None):
        """`shard=(rank, world)` (extension): this rank runs tiles rank, rank+world, ... of the flattened tile list and
        ONE all-gather of the per-rank prediction blocks (patchfusion_b200/parallel.py) precedes the deterministic
        stitch, so the canvas is bit-identical to the single-device one.  `group`: the process group of `world` ranks
        (default group if None).  shard=None reproduces the reference's single-device behaviour."""
        if mode == 'train':
            raise NotImplementedError('training is out of scope of the H100 hot-path build (SURVEY.md §2 rows 10,12)')
        if tile_cfg is None:
            tile_cfg = self.tile_cfg
        else:
            tile_cfg = self.prepare_tile_cfg(tile_cfg['image_raw_shape'], tile_cfg['patch_split_num'])
        assert image_hr.shape[0] == 1
        self._check_shard(shard, group)
        eng = self.engine()
        ph, pw = self.patch_process_shape
        plan_fn = None
        if shard is not None and self.shard_coarse == 'owner':
            from .parallel import tile_plan
            plan_fn = lambda n: tile_plan(n, shard[1], self.owner_cost_tiles)

        def compute(phase, img, geom, tiles, sh, plan):
            lr = eng.buf('in.image_lr', (1, 3, ph, pw), torch.float32)
            return self._compute_phase(eng, phase, lr, img, geom, tiles, process_num, sh, plan, group)

        # patchfusion.py:441-448: N // process_num calls of process_num random tiles
        n_calls = int(cai_mode[1:]) // process_num if cai_mode[0] == 'r' else 0
        depth = self._tiled_forward(eng, image_hr, tile_cfg, cai_mode, process_num, shard, group, n_calls, compute,
                                    image_lr=image_lr, plan_fn=plan_fn)
        return depth, {'rgb': image_lr, 'depth_pred': depth, 'depth_gt': depth_gt}
