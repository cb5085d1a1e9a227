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

from .params import FP8_LAYERS, ParamTree, _get, fusion_fp8_amax, fusion_precision, state_layout, synthetic_state_dict, relative_position_index, \
    vit_fp8_amax, vit_fp8_layers, vit_precision, dpt_fp8_amax, dpt_fp8_layers, dpt_precision

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
    configuration, `make_lr`, blend masks, CUDA-graph replay, and the tiled forward of a batch of images (regular passes
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
        align_corners=True resample, pf_crop_resize with one whole-image tile per image): [B,3,H,W] -> [B,3,ph,pw].
        A list of B images [1,3,H_b,W_b] of different sizes (a mixed batch) gives the same [B,3,ph,pw] batch, through
        pf_crop_resize_multi; every image must resize to the same (ph, pw)."""
        from . import ops
        if isinstance(image_hr, (list, tuple)):
            imgs = [x.float().contiguous() for x in image_hr]
            sizes = sorted({self.resizer.out_size(*x.shape[-2:]) for x in imgs})
            if len(sizes) != 1:
                raise ValueError('make_lr: the images resize to different sizes %s' % sizes)
            (ph, pw), B, dev = sizes[0], len(imgs), imgs[0].device
            out = torch.empty((B, 3, ph, pw), dtype=torch.float32, device=dev)
            table = torch.empty((ops.crop_table_bytes(B),), dtype=torch.uint8, device=dev)
            ops.crop_table(imgs, [tuple(x.shape[-2:]) for x in imgs], table)
            org = torch.zeros((B, 2), dtype=torch.int32, device=dev)
            ops.crop_resize_multi(table, org, torch.arange(B, dtype=torch.int32, device=dev), ph, pw, out)
            return out
        img = image_hr.float().contiguous()
        B = img.shape[0]
        H, W = img.shape[-2:]
        ph, pw = self.resizer.out_size(H, W)
        out = torch.empty((B, 3, ph, pw), dtype=torch.float32, device=img.device)
        org = torch.zeros((B, 2), dtype=torch.int32, device=img.device)
        index = torch.arange(B, dtype=torch.int32, device=img.device) if B > 1 else None
        ops.crop_resize(img, org, index, H, W, ph, pw, out)
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
            # thread-local capture: only this thread is barred from unsafe CUDA calls while it captures.  Other threads
            # keep working; Tester's PNG writer, for one, waits on the previous image's copy events while the next
            # image's forward captures its graphs.  In the default global mode that wait fails and invalidates the
            # capture.
            with torch.cuda.graph(g, capture_error_mode='thread_local'):
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

    def _stitch_phase(self, eng, phase, full, origins, slots, th, tw, mask, up, base, canvas, want, avg_out=None):
        """pf_stitch_gather of one image's tiles (deterministic order; tile i is row slots[i] of the gathered
        predictions `full`) -> requested canvases.  avg_out: the [CH, CW] tensor the average is written into."""
        from . import ops
        CH, CW = canvas
        n = len(origins)
        tab = eng.buf('stitch.tab.' + phase, (n, 3), torch.int32)
        tab.copy_(torch.tensor([(oy, ox, sl) for (oy, ox), sl in zip(origins, slots)], dtype=torch.int32))
        dev = full.device
        outs = {k: torch.empty((CH, CW), dtype=torch.float32, device=dev) for k in want if k != 'avg' or avg_out is None}
        if 'avg' in want and avg_out is not None:
            outs['avg'] = avg_out
        ops.call('pf_stitch_gather', full, tab, n, th, tw, mask, up[0], up[1],
                 base[0] if base else None, base[1] if base else None, CH, CW,
                 outs.get('num'), outs.get('den'), outs.get('avg'), ops.stream_ptr())
        return outs

    def _draw_random_boxes(self, n_calls, process_num, H, W, h, w, shard, group, dev, n_images=1):
        """draw_random_boxes for n_images images of one geometry, each with n_calls calls."""
        return TiledModel.draw_random_boxes([(n_calls, H, W, h, w)] * n_images, process_num, shard, group, dev)

    @staticmethod
    def draw_random_boxes(specs, process_num, shard, group, dev):
        """Random tiles (image, y, x), image by image, each in the reference's draw order (baseline_pretrain.py:155-156:
        process_num rows, then ONE shared column per call): the draws of B sequential single-image calls.  specs[b] =
        (calls, H, W, h, w) of image b (calls 0: the image has no random phase).  Under real sharding rank 0's draws
        are broadcast once for the batch so every rank stitches the same list (all ranks still advance their own
        `random` state identically)."""
        boxes = []
        for b, (n_calls, H, W, h, w) in enumerate(specs):
            for _ in range(n_calls):
                ys = [random.randint(0, H - h - 1) for _ in range(process_num)]
                x0 = random.randint(0, W - w - 1)
                boxes += [(b, y, x0) for y in ys]
        if shard is not None and shard[0] != 'emulate' and boxes:
            import torch.distributed as dist
            t = torch.tensor(boxes, dtype=torch.int32, device=dev if dist.get_backend(group) == 'nccl' else 'cpu')
            dist.broadcast(t, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
            boxes = [tuple(b) for b in t.cpu().tolist()]
        return boxes

    @staticmethod
    def batch_tiles(tiles, n_images):
        """The batch's tile list: every image's tiles (y, x) in their single-image order, image-major, as
        (image, y, x).  Tile i of image b is item b * len(tiles) + i."""
        return TiledModel.mixed_tiles([tiles] * n_images)

    @staticmethod
    def mixed_tiles(per_image):
        """The tile list of images with tile lists of their own (per_image[b]: image b's (y, x) tiles), image-major,
        as (image, y, x)."""
        return [(b, y, x) for b, tiles in enumerate(per_image) for (y, x) in tiles]

    @staticmethod
    def regular_tiles(tile_cfg, cai_mode, patch_process_shape):
        """One image's regular tiles in the reference's order (baseline_pretrain.py:221-251): raw (y, x) origins in the
        image and the matching proc origins on the patch_reensemble canvas.  m1: the split grid; m2 and rN add the
        three grids shifted by half a tile."""
        H, W = tile_cfg['image_raw_shape']
        h, w = tile_cfg['patch_raw_shape']
        ph, pw = patch_process_shape
        offsets = [((0, 0), (0, 0))]
        if cai_mode == 'm2' or cai_mode[0] == 'r':
            offsets += [((0, w // 2), (0, pw // 2)), ((h // 2, 0), (ph // 2, 0)), ((h // 2, w // 2), (ph // 2, pw // 2))]
        raw, proc = [], []
        for (oy, ox), (py, px) in offsets:
            assert ox >= 0 and oy >= 0
            ny, nx = (H - oy) // h, (W - ox) // w
            raw += [(h * a + oy, w * b + ox) for a in range(ny) for b in range(nx)]
            proc += [(ph * a + py, pw * b + px) for a in range(ny) for b in range(nx)]
        return raw, proc

    @staticmethod
    def is_mixed(geom):
        """geom is one (H, W, h, w, ph, pw) for the whole batch, or a tuple of them, one per image (a mixed batch)"""
        return isinstance(geom[0], tuple)

    @staticmethod
    def roi_boxes(items, geoms):
        """ROI boxes [n, 4] fp32 (x1, y1, x2, y2 in patch_process units) of (image, y, x) items, or (y, x) items of
        image 0, exactly as baseline_pretrain.py:268-282: the integer pixel box times its image's fp32 factors
        (geoms[b] = (H, W, h, w, ph, pw) of image b)."""
        fac = [(np.float32(1 / W * pw), np.float32(1 / H * ph), h, w) for (H, W, h, w, ph, pw) in geoms]
        out = np.empty((len(items), 4), dtype=np.float32)
        for i, it in enumerate(items):
            fx, fy, h, w = fac[it[0] if len(it) == 3 else 0]
            y, x = it[-2:]
            out[i] = (np.float32(x) * fx, np.float32(y) * fy, np.float32(x + w) * fx, np.float32(y + h) * fy)
        return out

    @staticmethod
    def _crop(img, geom, raw, tile_image, out):
        """crop + resize to out [T,3,ph,pw] of the tiles at origins `raw` ([T,2] int32) of the images tile_image ([T]
        int32, None: image 0).  One geometry: img is the batch [B,3,H,W] (or [3,H,W]).  Mixed batch: img is the
        pf_crop_resize_multi table of the images, which carries each image's size and tile size."""
        from . import ops
        if TiledModel.is_mixed(geom):
            ops.crop_resize_multi(img, raw, tile_image, out.shape[2], out.shape[3], out)
        else:
            H, W, h, w, ph, pw = geom
            ops.crop_resize(img, raw, tile_image, h, w, ph, pw, out)

    def _batch_inputs(self, image_hr, tile_cfg, cai_mode):
        """forward's image_hr / tile_cfg / cai_mode -> (image_hr, tile_cfg, cai_mode, mixed).  One geometry (a [B,3,H,W]
        tensor, a dict or None, a string): the tensor, the prepared tile_cfg and the mode, mixed False.  A mixed batch
        (any of the three a list; a tensor or a single tile_cfg / mode applies to every image): lists of B images
        [1,3,H_b,W_b], prepared tile_cfgs and modes, mixed True, after the reference's per-image checks.  A mixed batch
        whose images all share one tile_cfg and mode comes back as that tensor batch, still with mixed True (the caller
        returns a list)."""
        def prep(c):
            return self.tile_cfg if c is None else self.prepare_tile_cfg(c['image_raw_shape'], c['patch_split_num'])
        lists = [isinstance(a, (list, tuple)) for a in (image_hr, tile_cfg, cai_mode)]
        if not any(lists):
            return image_hr, prep(tile_cfg), cai_mode, False
        B = len(image_hr) if lists[0] else image_hr.shape[0]
        if B < 1:
            raise ValueError('a mixed batch needs at least one image')
        for a, is_list, name in ((tile_cfg, lists[1], 'tile_cfg'), (cai_mode, lists[2], 'cai_mode')):
            if is_list and len(a) != B:
                raise ValueError('%s holds %d entries for %d images' % (name, len(a), B))
        images = list(image_hr) if lists[0] else list(image_hr.split(1))
        cfgs = [prep(c) for c in (tile_cfg if lists[1] else [tile_cfg] * B)]
        modes = list(cai_mode) if lists[2] else [cai_mode] * B
        for x, cfg in zip(images, cfgs):
            assert x.dim() == 4 and x.shape[:2] == (1, 3), 'every image of a mixed batch must be [1, 3, H, W]'
            assert tuple(x.shape[-2:]) == tuple(cfg['image_raw_shape']), 'image_hr must already be at image_raw_shape'
        keys = {(tuple(c['image_raw_shape']), tuple(c['patch_split_num']), m) for c, m in zip(cfgs, modes)}
        if len(keys) == 1:
            return torch.cat(images), cfgs[0], modes[0], True
        return images, cfgs, modes, True

    @staticmethod
    def image_ranges(items, n_images):
        """[start, stop) of each image's items in an image-major list of (image, ...) items."""
        starts = [0] * (n_images + 1)
        for it in items:
            starts[it[0] + 1] += 1
        for b in range(n_images):
            starts[b + 1] += starts[b]
        return [(starts[b], starts[b + 1]) for b in range(n_images)]

    @staticmethod
    def split_tiles(tiles):
        """Tile list -> ([(y, x)], [image]).  Plain (y, x) tiles belong to image 0 (single-image callers)."""
        yx = [t[-2:] for t in tiles]
        return yx, [t[0] if len(t) == 3 else 0 for t in tiles]

    def _tiled_forward(self, eng, image_hr, tile_cfg, cai_mode, process_num, shard, group, n_random_calls, compute,
                       image_lr=None, plan_fn=None):
        """Tiled inference of a batch of B images: the regular passes (baseline_pretrain.py:221-331,
        patchfusion.py:417-439) are independent tiles whose stitch is a weighted sum, so all passes of all images are
        flattened into one ordered, image-major tile list of (image, y, x) and micro-batched (a micro-batch may mix
        images); rN modes then resize each canvas to image_raw_shape and add n_random_calls(mode) calls of
        `process_num` random tiles per image.  The stitch runs once per image over that image's part of the list, so
        image b's canvas equals its single-image run bit for bit.
        One geometry: image_hr [B,3,H,W], one prepared tile_cfg and mode -> depth [B,1,H',W'].  Mixed batch (see
        _batch_inputs): lists of B images [1,3,H_b,W_b], tile_cfgs and modes -> a list of B depths [1,1,H'_b,W'_b];
        each image gets its own static buffer and the crops read them through one pf_crop_resize_multi table.
        image_lr (PatchFusion) goes into its static buffer; plan_fn(n) gives the rank of each regular tile (None:
        round-robin)."""
        from . import ops
        from .parallel import slot_table
        mixed = isinstance(image_hr, list)
        B = len(image_hr) if mixed else image_hr.shape[0]
        cfgs = tile_cfg if mixed else [tile_cfg] * B
        modes = cai_mode if mixed else [cai_mode] * B
        dev = image_hr[0].device
        ph, pw = self.patch_process_shape
        geoms = [tuple(c['image_raw_shape']) + tuple(c['patch_raw_shape']) + (ph, pw) for c in cfgs]
        world = 1 if shard is None else shard[1]
        # inputs into static buffers (stable addresses for the captured graphs)
        if mixed:
            bufs = [eng.buf('in.image_hr.%d' % b, (1, 3) + g[:2], torch.float32) for b, g in enumerate(geoms)]
            for buf, x in zip(bufs, image_hr):
                assert tuple(x.shape[-2:]) == buf.shape[-2:], 'image_hr must already be at image_raw_shape'
                buf.copy_(x)
            img = ops.crop_table(bufs, [g[2:4] for g in geoms],
                                 eng.buf('in.crop_table', (ops.crop_table_bytes(B),), torch.uint8))
            geom = tuple(geoms)
        else:
            geom = geoms[0]
            assert tuple(image_hr.shape[-2:]) == geom[:2], 'image_hr must already be at image_raw_shape'
            img = eng.buf('in.image_hr', (B, 3) + geom[:2], torch.float32)
            img.copy_(image_hr)
        if image_lr is not None:
            assert image_lr.shape[0] == B, 'image_lr and image_hr must hold the same number of images'
            eng.buf('in.image_lr', (B, 3, ph, pw), torch.float32).copy_(image_lr)
        mask = self._mask((ph, pw), dev)
        raws, procs = zip(*[self.regular_tiles(c, m, (ph, pw)) for c, m in zip(cfgs, modes)])
        is_r = [m[0] == 'r' for m in modes]
        tiles = self.mixed_tiles(raws)
        plan = plan_fn(len(tiles)) if plan_fn is not None else None
        full = self._exchange(lambda sh: compute('reg', img, geom, tiles, sh, plan), shard, group)
        slots = slot_table(len(tiles), world, plan)
        sizes = [g[:2] if r else tuple(c['patch_reensemble_shape']) for g, c, r in zip(geoms, cfgs, is_r)]
        if mixed:
            depth = [torch.empty((1, 1) + s, dtype=torch.float32, device=dev) for s in sizes]
        else:
            depth = torch.empty((B, 1) + sizes[0], dtype=torch.float32, device=dev)
        canvas = [d[0] for d in depth] if not mixed else [d[0, 0] for d in depth]      # image b's [H', W'] output
        bases = [None] * B
        for b, (i0, i1) in enumerate(self.image_ranges(tiles, B)):
            H, W = geoms[b][:2]
            RH, RW = cfgs[b]['patch_reensemble_shape']
            outs = self._stitch_phase(eng, 'reg', full, procs[b], slots[i0:i1], ph, pw, mask, (0, 0), None,
                                      (RH, RW), ('num', 'den') if is_r[b] else ('avg',), avg_out=canvas[b])
            if is_r[b]:
                n2 = torch.empty((H, W), dtype=torch.float32, device=dev)
                d2 = torch.empty_like(n2)
                ops.call('pf_stitch_resize', outs['num'], outs['den'], RH, RW, H, W, n2, d2, ops.stream_ptr())
                bases[b] = (n2, d2)
        if not any(is_r):
            return depth
        specs = [(n_random_calls(m) if r else 0,) + g[:4] for m, r, g in zip(modes, is_r, geoms)]
        boxes = self.draw_random_boxes(specs, process_num, shard, group, dev)
        ranges = self.image_ranges(boxes, B)
        for b in range(B):
            if is_r[b] and ranges[b][0] == ranges[b][1]:        # rN with no random call: the resized canvas
                torch.div(bases[b][0], bases[b][1], out=canvas[b])
        for s0, s1 in self._chunks(len(boxes), self.random_chunk):
            part = boxes[s0:s1]
            full = self._exchange(lambda sh: compute('rnd', img, geom, part, sh, None), shard, group)
            slots = slot_table(len(part), world)
            for b, (i0, i1) in enumerate(self.image_ranges(part, B)):
                if i0 == i1:
                    continue
                H, W, h, w = geoms[b][:4]
                last = s0 + i1 == ranges[b][1]
                outs = self._stitch_phase(eng, 'rnd', full, [t[1:] for t in part[i0:i1]], slots[i0:i1], ph, pw,
                                          self._mask((h, w), dev), (h, w), bases[b], (H, W),
                                          ('avg',) if last else ('num', 'den'), avg_out=canvas[b])
                if not last:
                    bases[b] = (outs['num'], outs['den'])
        return depth


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
        self.fusion_precision = fusion_precision(config)     # ValueError on anything but 'bf16' / 'fp8' / 'fp8_static'
        fusion_fp8_amax(config)                              # ValueError on a malformed calibration table
        for br in (config.coarse_branch, config.fine_branch):
            if br.type not in ('ZoeDepth', 'DA-ZoeDepth'):
                raise NotImplementedError
        self.resizer = Resize(config.patch_process_shape[1], config.patch_process_shape[0])
        self.vit_precision = vit_precision(config)           # ValueError on anything but 'bf16' / 'fp8_static'
        vit_fp8_amax(config)                                 # ValueError on a malformed ViT calibration table
        self.dpt_precision = dpt_precision(config)           # ValueError on anything but 'bf16' / 'fp8_static'
        dpt_fp8_amax(config)                                 # ValueError on a malformed DPT calibration table
        self._build_tree(state_layout(config))      # raises ValueError / NotImplementedError like the reference
        self.consistency_training = False
        self._runtime_init()
        self._coarse = None
        # coarse branch + G2L (batch B) on a side stream next to the first fine branch: measured in DESIGN.md
        self.overlap_coarse = os.environ.get('PF_B200_OVERLAP_COARSE', '1') != '0'
        self._side_stream = None
        # tile-sharded forward: 'owner' = rank b % world computes image b's coarse branch + G2L, takes
        # `owner_cost_tiles` fewer tiles per image it owns, and one all-gather of the packed results reaches every
        # rank; 'replicate' = every rank computes all of them (no exchange)
        self.shard_coarse = os.environ.get('PF_B200_SHARD_COARSE', 'owner')
        self.owner_cost_tiles = float(os.environ.get('PF_B200_OWNER_COST', '2.7'))
        self._pack = None
        self._items = None
        self._local_coarse = {}
        self._pending_fine = {}
        self._coarse_src = 'local'
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
        else:
            # the calibration tables are part of the config: a changed table re-points the stage and drops the graphs
            # captured with the old scales
            if self._engine.fp8_static:
                table = fusion_fp8_amax(self.config)
                if table != self._engine.fp8_amax:
                    self._engine.set_fp8_amax(table)
                    self._graphs = {}
            if self._engine.vit_fp8_static:
                table = vit_fp8_amax(self.config)
                if table != self._engine.vit_amax:
                    self._engine.set_vit_fp8_amax(table)
                    self._graphs = {}
            if self._engine.dpt_fp8_static:
                table = dpt_fp8_amax(self.config)
                if table != self._engine.dpt_amax:
                    self._engine.set_dpt_fp8_amax(table)
                    self._graphs = {}
        return self._engine

    @torch.no_grad()
    def calibrate_fp8(self, image_lr, image_hr, cai_mode='m1', process_num=4, tile_cfg=None, reset=False):
        """Post-training calibration of the static FP8 U-Net ('fp8' and 'fp8_static' models), of the 'fp8_static'
        ViT encoders and of the 'fp8_static' DPT decoders: runs forward(mode='infer') on the given images (the same
        arguments: batches, mixed geometry, rN modes drawing from `random`) with the per-tile 'fp8' U-Net arithmetic and
        the bf16 branches on this model's panels, and takes, for each of the 34 FP8 convs, each E4M3 ViT linear and each
        E4M3 DPT conv, the maximum over all tiles and images of its input's amax.  Each table is merged by max into
        config['fusion_fp8_amax'] / config['vit_fp8_amax'] / config['dpt_fp8_amax'] (reset=True starts from empty
        tables), which 'fp8_static' then runs with.  Returns the U-Net table, else the ViT table, else the DPT table.
        Runs eagerly: no graph of it is kept, and the graphs of earlier forwards are dropped."""
        unet = self.fusion_precision in ('fp8', 'fp8_static')
        vit = self.vit_precision == 'fp8_static'
        dpt = self.dpt_precision == 'fp8_static'
        if not unet and not vit and not dpt:
            raise ValueError("calibrate_fp8 needs fusion_precision 'fp8' or 'fp8_static', vit_precision 'fp8_static' or "
                             "dpt_precision 'fp8_static' (this model: %r, %r, %r)"
                             % (self.fusion_precision, self.vit_precision, self.dpt_precision))
        eng = self.engine()
        eng.calib = {}
        graphs, self.use_cuda_graphs = self.use_cuda_graphs, False
        try:
            self.forward('infer', image_lr, image_hr, tile_cfg=tile_cfg, cai_mode=cai_mode, process_num=process_num)
            found = {k: v.item() for k, v in eng.calib.items()}
        finally:
            eng.calib = None
            self.use_cuda_graphs = graphs
            self._graphs = {}
        hub = getattr(self, '_hub_mixin_config', None)
        for on, key, names, check in ((unet, 'fusion_fp8_amax', FP8_LAYERS, fusion_fp8_amax),
                                      (vit, 'vit_fp8_amax', vit_fp8_layers(self.config), vit_fp8_amax),
                                      (dpt, 'dpt_fp8_amax', dpt_fp8_layers(self.config), dpt_fp8_amax)):
            if not on:
                continue
            missing = [k for k in names if k not in found]
            if missing:
                raise RuntimeError('calibrate_fp8: no input amax for %s (a conv read through PF_OPT_FUSED_RESAMPLE has '
                                   'no materialised input to measure)' % missing)
            table = {} if reset else dict(check(self.config) or {})
            for k in names:
                table[k] = max(table.get(k, 0.0), found[k]) if found[k] == found[k] else found[k]
            self.config[key] = check({key: table, 'coarse_branch': self.config.coarse_branch,
                                      'fine_branch': self.config.fine_branch})     # ValueError on NaN / inf
            if isinstance(hub, dict):               # the config save_pretrained writes
                hub[key] = dict(self.config[key])
        self.engine()
        return dict(self.config['fusion_fp8_amax' if unet else ('vit_fp8_amax' if vit else 'dpt_fp8_amax')])

    def invalidate(self):
        super().invalidate()
        self._pack = self._items = None
        self._local_coarse = {}

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
    def _coarse_stage(self, eng, lr, pack=None):
        """coarse branch + G2L of the images `lr` [k,3,ph,pw], at batch k.  pack (tile-sharded owner): this rank's
        pack views (see _ensure_pack); the results are copied into its first k images, for the all-gather."""
        cd, cf = eng.branch('coarse', lr)
        res = (cd, cf, eng.g2l(cf))
        if pack is None:
            # a replayed graph does not run this method: _compute_phase restores the views of this batch size
            self._coarse = self._local_coarse[lr.shape[0]] = res
            return
        k = lr.shape[0]
        pack[0][:k].copy_(res[0])
        for d, m in zip(pack[1] + pack[2], res[1] + res[2]):
            d.t[:k].copy_(m.t)

    def _coarse_items(self, eng, lr):
        """(shape of one image, dtype, logical channels or None) of the 13 coarse results: coarse depth fp32, 6 coarse
        maps, 6 G2L maps.  They follow from the model geometry alone; the first call runs the coarse stage once on one
        image to read them off the stage outputs (every rank, outside any timed region)."""
        if getattr(self, '_items', None) is None or self._items[1] is not eng:
            cd, cf = eng.branch('coarse', lr[:1])
            g2l = eng.g2l(cf)
            items = [(tuple(cd.shape[1:]), torch.float32, None)] + \
                [(tuple(m.t.shape[1:]), m.t.dtype, m.C) for m in cf + g2l]
            self._items = (items, eng)
        return self._items[0]

    def _ensure_pack(self, eng, lr, kmax, world):
        """Buffers of the coarse-owner exchange for ranks that own up to `kmax` images each: this rank's pack (the 13
        results of kmax images in 256-B aligned segments) and the [world, pack] all-gather destination.  Returns
        (pack bytes, pack views, gathered bytes, per-rank views into the gathered buffer)."""
        key = (eng, kmax, world)
        if self._pack is not None and self._pack[0] == key:
            return self._pack[1]
        from .engine import Map
        items = self._coarse_items(eng, lr)
        offs, total = [], 0
        for shape, dt, _ in items:
            offs.append(total)
            total += (kmax * int(np.prod(shape)) * torch.empty((), dtype=dt).element_size() + 255) // 256 * 256

        def views(buf):
            out = []
            for (shape, dt, C), o in zip(items, offs):
                nb = kmax * int(np.prod(shape)) * torch.empty((), dtype=dt).element_size()
                t = buf[o:o + nb].view(dt).view((kmax,) + tuple(shape))
                out.append(t if C is None else Map(t, C))
            return out[0], out[1:7], out[7:]
        pack = eng.buf('coarse.pack', (total,), torch.uint8)
        gathered = eng.buf('coarse.gathered', (world, total), torch.uint8)
        res = (pack, views(pack), gathered, [views(gathered[r]) for r in range(world)])
        self._pack = (key, res)
        return res

    def _batch_coarse(self, eng, lr, B):
        """The batch-B coarse results every fusion of a tile-sharded owner-mode forward reads (the all-gathered packs
        are copied into them image by image)."""
        from .engine import Map
        items = self._coarse_items(eng, lr)
        out = []
        for i, (shape, dt, C) in enumerate(items):
            t = eng.buf('coarse.batch.%d' % i, (B,) + tuple(shape), dt)
            out.append(t if C is None else Map(t, C))
        return out[0], out[1:7], out[7:]

    def _exchange_coarse(self, eng, lr, B, rank, world, group, real):
        """Coarse-owner mode: image b's coarse branch + G2L run on rank b % world, at the batch of that rank's images;
        every rank packs its results and ONE all-gather of the equal-size packs gives everybody all B images, which
        are unpacked into the batch-B coarse buffers.  Emulated sharding runs every rank's coarse stage here, at the
        first rank computed."""
        from .parallel import coarse_owners, unpack_owned
        owners = coarse_owners(B, world)
        kmax = -(-B // world)
        pack, pviews, gathered, gviews = self._ensure_pack(eng, lr, kmax, world)
        geom = tuple(lr.shape)
        for r in (range(world) if not real else [rank]):
            mine = [b for b in range(B) if owners[b] == r]
            if not mine:
                continue
            lr_r = eng.buf('in.image_lr.owned', (len(mine),) + tuple(lr.shape[1:]), torch.float32)

            def stage(mine=mine, lr_r=lr_r):
                for j, b in enumerate(mine):
                    lr_r[j].copy_(lr[b])
                self._coarse_stage(eng, lr_r, pack=pviews)
            self._graphed(('coarse.pack', tuple(mine), kmax, B, r, world) + geom, stage)
            if not real:
                gathered[r].copy_(pack)
        if real:
            self._gather_packs(pack, gathered, group)
        batch = self._batch_coarse(eng, lr, B)
        unpack_owned(batch[0], [g[0] for g in gviews], world)
        for i in range(6):
            unpack_owned(batch[1][i].t, [g[1][i].t for g in gviews], world)
            unpack_owned(batch[2][i].t, [g[2][i].t for g in gviews], world)
        self._coarse = batch

    @staticmethod
    def _gather_packs(pack, gathered, group):
        import torch.distributed as dist
        if dist.get_backend(group) == 'nccl':
            dist.all_gather_into_tensor(gathered.view(-1), pack, group=group)
        else:                                   # gloo: list form
            dist.all_gather(list(gathered.unbind(0)), pack, group=group)

    def _fine_stage(self, eng, img, T, geom, raw, tile_image=None):
        """crop+resize -> fine branch for the T tiles whose raw origins are the device rows `raw` ([T,2] int32) of the
        images tile_image ([T] int32, None: image 0) of img ([B,3,H,W] or [3,H,W], or a mixed batch's crop table)."""
        ph, pw = self.patch_process_shape
        crops = eng.buf('tile.crops', (T, 3, ph, pw), torch.float32)
        self._crop(img, geom, raw, tile_image, crops)
        # ONE arena for the tile stages, sized for the largest micro-batch: [fine branch | fusion]
        nb = (eng.branch_bytes('fine', T) + 255) // 256 * 256
        arena = eng.arena('tile', nb + eng.fusion_bytes(T, self._coarse[2]))
        fd, ff = eng.branch('fine', crops, ws=(arena, 0))
        return crops, fd, ff, (arena, nb)

    def _fusion_stage(self, eng, fine, boxes, out, tile_image=None):
        """guided fusion of one micro-batch; the fused depth goes straight into its rows `out` of the prediction block.
        tile_image: the image of the batch-B coarse results each tile reads (None: image 0)."""
        cd, cf, g2l = self._coarse
        crops, fd, ff, ws = fine
        eng.fusion(crops, boxes, fd, ff, cd, cf, g2l, depth_out=out, ws=ws, tile_image=tile_image)

    def _image_stage(self, eng, lr, img, geom, sizes, io_raw, io_box, io_img, blk, with_coarse, part='all'):
        """The static kernel sequence of one phase of the batch on this rank: [coarse branch + G2L of the B images]
        and the micro-batches (fine branch + fusion each; a micro-batch may mix images, io_img gives each tile's).
        The coarse stage has no dependency on the first fine branch, so it runs on a side stream next to it (its
        whole-image kernels fill a fraction of the SMs).
        part='pre' / 'post' (tile-sharded, ranks that own no coarse stage): the fine branch of the first micro-batch
        runs BEFORE the all-gather of the owners' coarse results arrives, everything else after it."""
        from . import lib
        ti = (lambda s0, s1: None) if io_img is None else (lambda s0, s1: io_img[s0:s1])
        # the fine outputs of 'pre' are views whose addresses depend on its micro-batch size only: kept per size, so a
        # 'post' captured after a replayed 'pre' (which runs no Python) reads the right ones
        if part == 'pre':
            self._pending_fine[sizes[0]] = self._fine_stage(eng, img, sizes[0], geom, io_raw[:sizes[0]], ti(0, sizes[0]))
            return
        s0 = 0
        if part == 'post':
            T0 = sizes[0]
            self._fusion_stage(eng, self._pending_fine[T0], io_box[:T0], blk[:T0], ti(0, T0))
            s0, sizes = T0, sizes[1:]
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
        for T in sizes:
            fine = self._fine_stage(eng, img, T, geom, io_raw[s0:s0 + T], ti(s0, s0 + T))
            if side is not None:
                cur.wait_stream(side)
                side = None
            self._fusion_stage(eng, fine, io_box[s0:s0 + T], blk[s0:s0 + T], ti(s0, s0 + T))
            s0 += T

    def _compute_phase(self, eng, phase, lr, img, geom, raw, process_num, shard, plan=None, group=None):
        """Fused predictions of this rank's tiles of the (global, ordered) tile list `raw` ((image, y, x) items) ->
        its block [block_rows, ph, pw] fp32 (row j = the j-th tile of the list that `plan` gives to this rank).
        geom: one (H, W, h, w, ph, pw), or one per image of a mixed batch (img is then its crop table)."""
        from .parallel import shard_indices, block_rows
        ph, pw = self.patch_process_shape
        mixed = self.is_mixed(geom)
        rank, world = (0, 1) if shard is None else shard
        B = lr.shape[0]
        n = len(raw)
        own = shard_indices(n, rank, world, plan)
        blk = eng.buf('pred.blk.' + phase, (block_rows(n, world, plan), ph, pw), torch.float32)
        with_coarse = phase == 'reg'
        owner_mode = with_coarse and shard is not None and self.shard_coarse == 'owner'
        real = shard is not None and self._real_shard
        owns_coarse = owner_mode and rank < B               # image b's coarse stage runs on rank b % world
        split = owner_mode and real and not owns_coarse and bool(own)
        if with_coarse and not owner_mode:
            # the views the coarse stage of this batch size last produced: valid whenever its graph is (both are
            # renewed when a workspace moves), and what the later 'rnd' phase of this forward reads
            self._coarse = self._local_coarse.get(B, self._coarse)
        if owner_mode:
            with_coarse = False
            if split:
                self._coarse = self._batch_coarse(eng, lr, B)   # shapes for the 'pre' stage; filled by the exchange
            elif real or rank == 0:                             # emulated ranks run in order: rank 0 does them all
                self._exchange_coarse(eng, lr, B, rank, world, group, real)
        if not own:
            return blk
        io_raw = eng.buf('io.raw.' + phase, (len(own), 2), torch.int32)
        io_box = eng.buf('io.box.' + phase, (len(own), 4), torch.float32)
        items = [raw[i] for i in own]
        chunk, images = self.split_tiles(items)
        io_raw.copy_(torch.tensor(chunk, dtype=torch.int32))
        io_img = None
        if B > 1 or mixed:
            io_img = eng.buf('io.img.' + phase, (len(own),), torch.int32)
            io_img.copy_(torch.tensor(images, dtype=torch.int32))
        io_box.copy_(torch.from_numpy(self.roi_boxes(items, geom if mixed else [geom] * B)))
        sizes = self._micro_sizes(len(own), process_num)
        # a mixed batch's key holds every image's geometry; the modes only change tile counts, which `sizes` holds
        key = ('image', phase, tuple(sizes), blk.shape[0], with_coarse, B, self._coarse_src) + tuple(geom)
        run = lambda part: self._graphed(key + (part,), lambda: self._image_stage(
            eng, lr, img, geom, sizes, io_raw, io_box, io_img, blk, with_coarse, part))
        if split:
            run('pre')
            self._exchange_coarse(eng, lr, B, rank, world, group, real)
            run('post')
        else:
            run('all')
        return blk

    @torch.no_grad()
    def forward(self, mode, image_lr, image_hr, depth_gt=None, crops_image_hr=None, crop_depths=None, bboxs=None,
                tile_cfg=None, cai_mode='m1', process_num=4, shard=None, group=None):
        """image_lr [B,3,ph,pw], image_hr [B,3,H,W] -> depth [B,1,H',W'] (extension: the reference takes B = 1).  All B
        images share tile_cfg, cai_mode and process_num; their tiles form one image-major list that is micro-batched
        and sharded together, the coarse branch + G2L run once at batch B, and image b's output equals, bit for bit,
        the single-image call on it made after images 0..b-1 from the same `random` state.
        `shard=(rank, world)` (extension): this rank runs its share of the flattened tile list and ONE all-gather of
        the per-rank prediction blocks (patchfusion_b200/parallel.py) precedes the deterministic stitch, so the canvas
        is bit-identical to the single-device one.  `group`: the process group of `world` ranks (default group if
        None).  shard=None reproduces the reference's single-device behaviour.
        Mixed batch (extension): image_hr a list of B images [1,3,H_b,W_b], each at its own image_raw_shape, tile_cfg a
        list of B dicts and cai_mode a string or a list of B modes; process_num is shared.  image_lr stays
        [B,3,ph,pw].  Returns a list of B depths [1,1,H'_b,W'_b] (info['depth_pred'] is that list) under the same
        contract: image b equals the single-image call on it made after images 0..b-1."""
        if mode == 'train':
            raise NotImplementedError('training is out of scope of the H100 hot-path build (SURVEY.md §2 rows 10,12)')
        image_hr, tile_cfg, cai_mode, as_list = self._batch_inputs(image_hr, tile_cfg, cai_mode)
        B = len(image_hr) if isinstance(image_hr, list) else image_hr.shape[0]
        assert B >= 1 and image_lr.shape[0] == B, 'image_lr and image_hr must hold the same number (>= 1) of images'
        self._check_shard(shard, group)
        eng = self.engine()
        eng._fusion_struct()            # 'fp8_static' without a calibration table: RuntimeError naming calibrate_fp8
        ph, pw = self.patch_process_shape
        plan_fn = None
        owner = shard is not None and self.shard_coarse == 'owner'
        self._coarse_src = 'gathered' if owner else 'local'
        if owner:
            from .parallel import tile_plan
            plan_fn = lambda n: tile_plan(n, shard[1], self.owner_cost_tiles, images=B)

        def compute(phase, img, geom, tiles, sh, plan):
            lr = eng.buf('in.image_lr', (B, 3, ph, pw), torch.float32)
            return self._compute_phase(eng, phase, lr, img, geom, tiles, process_num, sh, plan, group)

        # patchfusion.py:441-448: N // process_num calls of process_num random tiles
        n_calls = lambda m: int(m[1:]) // process_num
        depth = self._tiled_forward(eng, image_hr, tile_cfg, cai_mode, process_num, shard, group, n_calls, compute,
                                    image_lr=image_lr, plan_fn=plan_fn)
        if as_list and not isinstance(depth, list):
            depth = list(depth.split(1))
        return depth, {'rgb': image_lr, 'depth_pred': depth, 'depth_gt': depth_gt}
