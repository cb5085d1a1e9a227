"""Evaluation datasets with the reference's constructors and registry names: `UnrealStereo4kDataset`
(`estimator/datasets/u4k_dataset.py:20-259`, `mode='infer'` only) and `ImageDataset`
(`estimator/datasets/general_dataset.py:145-230`).

`dataset[i]` returns the image's host-side raw sources, not fp32 tensors: the uint8 frame (raw U4K bytes, or the
decoded image), the fp32 / uint16 ground-truth source map and its constants.  `prepare(sample, device)` copies those
bytes to the device and runs pf_ingest_raw_u8 / pf_ingest_u8 and pf_gt_prepare there, which yields the sample dict
`Tester.run` accepts (`image_hr`, `depth_gt`, `boundary`, `img_file_basename`).  The reference instead converts the
25 MB frame to fp32 (99.5 MB), divides the 8.3 MP disparity, runs get_boundaries and copies ~165 MB per 4K image.
`PreparedSamples` reads image i + 1 on a bounded reader thread (the reference's `num_workers`) into a fixed ring of
pinned buffers while image i computes.

`host_ground_truth` / `host_prepare` restate the reference's numpy preparation; they are the baseline the GPU path is
compared against, bit for bit."""
import os
import os.path as osp
import queue
import re
import threading
from collections import OrderedDict

import numpy as np
import torch

from . import imageio, metrics as pf_metrics

METRIC_KEYS = pf_metrics.KEYS + ('see',)
CITYSCAPES_FACTOR = 0.209313 * 2262.52         # general_dataset.py:129, baseline x focal length
ETH3D_SHAPE = (4032, 6048)                     # general_dataset.py:89
U4K_SHAPE = (2160, 3840)                       # u4k_dataset.py:115, general_dataset.py:24


def _check_resize_mode(resize_mode):
    """The dataset's resize_mode picks how the reference resizes image_lr.  Here image_lr is always the model's own
    (`model.make_lr`, the 'depth-anything' resize to patch_process_shape), so any other mode would silently give a
    different coarse input than the reference: 'zoe' (a 384 x 512, multiple-of-32 resize) raises."""
    if resize_mode != 'depth-anything':
        raise NotImplementedError(
            "resize_mode=%r: image_lr is computed by model.make_lr, which matches only resize_mode='depth-anything'.  "
            "The reference's _base_/datasets/u4k.py leaves test_in/test_out at 'zoe'; with a Depth-Anything config "
            "pass e.g. --cfg-options test_in_dataloader.dataset.resize_mode=depth-anything" % (resize_mode,))


def read_pfm(path):
    """`estimator/datasets/utils.py:readPFM`: (data [H,W] or [H,W,3] flipped upright, scale)."""
    with open(path, 'rb') as f:
        header = f.readline().rstrip().decode('utf-8')
        if header not in ('PF', 'Pf'):
            raise ValueError('%s: not a PFM file' % path)
        m = re.match(r'^(\d+)\s(\d+)\s$', f.readline().decode('utf-8'))
        if not m:
            raise ValueError('%s: malformed PFM header' % path)
        width, height = map(int, m.groups())
        scale = float(f.readline().rstrip().decode('utf-8'))
        endian = '<' if scale < 0 else '>'
        data = np.fromfile(f, endian + 'f')
    shape = (height, width, 3) if header == 'PF' else (height, width)
    return np.flipud(np.reshape(data, shape)), abs(scale)


def read_mid_calib(path):
    """Middlebury calib.txt -> (depth factor = baseline * f, doffs) (general_dataset.py:100-108)."""
    with open(path, 'r') as f:
        lines = f.readlines()
    focal = float(lines[0].strip().split(' ')[0].split('[')[1])
    base = float(lines[3].strip().split('=')[1])
    doffs = float(lines[2].strip().split('=')[1])
    return base * focal, doffs


class _EvalDataset:
    """Metrics and summary shared by both datasets (u4k_dataset.py:185-259)."""

    def get_metrics(self, depth_gt, result, disp_gt_edges, **kwargs):
        return pf_metrics.compute_metrics(depth_gt, result, disp_gt_edges=disp_gt_edges, min_depth_eval=self.min_depth,
                                          max_depth_eval=self.max_depth)

    @staticmethod
    def evaluate(results):
        """u4k_dataset.py:188-213: nanmean over the images of each metric, in the reference's order."""
        cols = list(zip(*[tuple(r.values()) for r in results]))
        return OrderedDict((k, float(np.nanmean(cols[i]))) for i, k in enumerate(METRIC_KEYS[:len(cols)]))

    @staticmethod
    def prepare(sample, device):
        return prepare(sample, device)


class UnrealStereo4kDataset(_EvalDataset):
    def __init__(self, mode, data_root, split, transform_cfg, min_depth, max_depth, patch_raw_shape=(540, 960),
                 resize_mode='zoe'):
        if mode != 'infer':
            raise NotImplementedError("UnrealStereo4kDataset mode=%r: only mode='infer' (evaluation) is built" % mode)
        _check_resize_mode(resize_mode)
        self.dataset_name = 'u4k'
        self.mode, self.data_root, self.split = mode, data_root, split
        self.data_infos = self.load_data_list()
        self.min_depth, self.max_depth = min_depth, max_depth
        self.patch_raw_shape = patch_raw_shape
        self.transform_cfg = transform_cfg

    def load_data_list(self):
        """Split lines `img_l img_r disp_l disp_r` (u4k_dataset.py:58-107): the left image as .raw, the depth factor
        baseline * f from the Extrinsics0/1 files next to the disparity, sorted by image path."""
        if self.split is None:
            raise NotImplementedError('UnrealStereo4kDataset needs a split file')
        infos = []
        with open(self.split) as f:
            for line in f:
                img_l, _, disp_l, _ = line.strip().split(' ')
                img_l = img_l[:-3] + 'raw'
                info = dict(depth_map_path=osp.join(self.data_root, disp_l), img_path=osp.join(self.data_root, img_l),
                            filename=img_l)
                disp_path = info['depth_map_path']
                with open(disp_path.replace('Disp0', 'Extrinsics0').replace('npy', 'txt')) as fe:
                    ext_l = fe.readlines()
                with open(disp_path.replace('Disp0', 'Extrinsics1').replace('npy', 'txt')) as fe:
                    ext_r = fe.readlines()
                focal = float(ext_l[0].split(' ')[0])
                info['focal'] = focal
                info['depth_factor'] = abs(float(ext_l[1].split(' ')[3]) - float(ext_r[1].split(' ')[3])) * focal
                infos.append(info)
        return sorted(infos, key=lambda x: x['img_path'])

    @staticmethod
    def basename(filename):
        """u4k_dataset.py:145-146, the leading character of the joined name dropped."""
        return osp.splitext(filename)[0].replace('/', '_')[1:]

    def __len__(self):
        return len(self.data_infos)

    def __getitem__(self, idx):
        info = self.data_infos[idx]
        return dict(image=np.fromfile(info['img_path'], dtype=np.uint8).reshape(U4K_SHAPE + (3,)), image_resize=None,
                    gt=np.load(info['depth_map_path'], mmap_mode='c').astype(np.float32, copy=False), gt_kind='u4k',
                    factor=info['depth_factor'], doffs=0.0, img_file_basename=self.basename(info['filename']))


class ImageDataset(_EvalDataset):
    def __init__(self, rgb_image_dir, mode='', min_depth=1e-3, max_depth=80, gt_dir=None, image_resolution=[2160, 3840],
                 dataset_name='', network_process_size=(384, 512), resize_mode='zoe'):
        _check_resize_mode(resize_mode)
        self.min_depth, self.max_depth, self.mode = min_depth, max_depth, mode
        self.rgb_image_dir = rgb_image_dir
        self.files = sorted(os.listdir(rgb_image_dir))
        self.gt_dir = gt_dir
        self.dataset_name = dataset_name
        if gt_dir is not None:
            self.gt_files = sorted(os.listdir(gt_dir))      # paired with self.files by sorted position
        self.image_resolution = image_resolution

    def __len__(self):
        return len(self.files)

    @staticmethod
    def image_name(name):
        return name.replace('.jpg', '').replace('.png', '').replace('.jpeg', '')

    def read_image(self, path):
        """(uint8 HxWx3 BGR, resize target or None) (general_dataset.py:22-47): U4K raw frames and Cityscapes images
        keep their size; every other image is resized bicubically to image_resolution."""
        import cv2
        if self.dataset_name == 'u4k':
            return np.fromfile(path, dtype=np.uint8).reshape(U4K_SHAPE + (3,)), None
        img = cv2.imread(path)              # IMREAD_COLOR: grey images arrive as 3-channel BGR
        if img is None:
            raise FileNotFoundError(path)
        if self.dataset_name == 'cityscapes':
            return img, None
        return img, tuple(int(v) for v in self.image_resolution)

    def read_ground_truth(self, path):
        """(source map, kind, factor, doffs) of general_dataset.py:60-139."""
        import cv2
        name = self.dataset_name
        if name == 'u4k':
            with open(path.replace('val_gt', 'val_factor').replace('.npy', '.txt')) as f:
                factor = float(f.readline())
            return np.load(path, mmap_mode='c').astype(np.float32, copy=False), 'u4k', factor, 0.0
        if name == 'gta':
            raise NotImplementedError('gta ground truth is read with the imageio package, which is not available here')
        if name == 'eth3d':
            return np.fromfile(path, dtype=np.float32).reshape(ETH3D_SHAPE), 'eth3d', 0.0, 0.0
        if name == 'mid':
            factor, doffs = read_mid_calib(path.replace('gts', 'calibs').replace('.pfm', '.txt'))
            return np.ascontiguousarray(read_pfm(path)[0], dtype=np.float32), 'mid', factor, doffs
        if name == 'cityscapes':
            d = cv2.imread(path, cv2.IMREAD_UNCHANGED)
            if d is None:
                raise FileNotFoundError(path)
            return d.astype(np.uint16, copy=False), 'cityscapes', CITYSCAPES_FACTOR, 0.0
        raise NotImplementedError('ground truth of dataset_name %r' % (name,))

    def __getitem__(self, index):
        image, resize = self.read_image(osp.join(self.rgb_image_dir, self.files[index]))
        s = dict(image=image, image_resize=resize, gt=None, gt_kind=None, factor=0.0, doffs=0.0,
                 img_file_basename=self.image_name(self.files[index]))
        if self.gt_dir is not None:
            s['gt'], s['gt_kind'], s['factor'], s['doffs'] = self.read_ground_truth(
                osp.join(self.gt_dir, self.gt_files[index]))
        return s


# ---------------------------------------------------------------------------------------------- device preparation
def prepare(sample, device):
    """Host sample -> the dict Tester.run takes, computed on `device`: image_hr (1,3,H,W) fp32 RGB, and with ground
    truth depth_gt (1,1,H,W) fp32 and boundary (1,1,H,W) uint8."""
    image = torch.as_tensor(sample['image']).to(device, non_blocking=True)
    if sample['image_resize'] is None:
        image_hr = imageio.ingest_raw(image, bgr=True)
    else:
        image_hr = imageio.ingest(image, sample['image_resize'], device, bgr=True)
    out = dict(image_hr=image_hr, img_file_basename=sample['img_file_basename'])
    if sample.get('gt') is not None:
        src = torch.as_tensor(sample['gt']).to(device, non_blocking=True)
        out['depth_gt'], out['boundary'] = imageio.gt_prepare(src, sample['gt_kind'], sample['factor'], sample['doffs'])
    return out


def _put(q, stop, item):
    """q.put that gives up once `stop` is set (the consumer has gone); returns False then."""
    while not stop.is_set():
        try:
            q.put(item, timeout=0.1)
            return True
        except queue.Full:
            pass
    return False


def _get(q, stop, poll=None):
    """q.get that gives up once `stop` is set; calls `poll` while it waits."""
    while not stop.is_set():
        try:
            return q.get(timeout=0.01)
        except queue.Empty:
            if poll is not None:
                poll()
    return None


class _PinnedRing:
    """A fixed set of pinned host buffers for the samples' arrays, allocated once, on the consumer's thread, before
    the reader starts: the reader thread then only copies bytes into a free slot and makes no CUDA call (pinning
    there would call cudaHostAlloc while the consumer may be capturing a CUDA graph).  A slot is handed back once the
    device copies made from it have completed.  Each slot holds a sample as large as the first one; a larger sample
    travels unpinned (a synchronous copy, same bytes)."""

    ALIGN = 256

    def __init__(self, first, slots):
        self.nbytes = sum(self._span(v) for v in first.values() if isinstance(v, np.ndarray))
        self.bufs = [torch.empty(max(self.nbytes, 1), dtype=torch.uint8, pin_memory=True) for _ in range(slots)]
        self.free = queue.Queue()
        for k in range(slots):
            self.free.put(k)

    def _span(self, v):
        return -(-v.nbytes // self.ALIGN) * self.ALIGN

    def fill(self, slot, sample):
        """sample with its arrays copied into slot `slot` (as tensors viewing it), or None when they do not fit"""
        if sum(self._span(v) for v in sample.values() if isinstance(v, np.ndarray)) > self.nbytes:
            return None
        out, off, buf = dict(sample), 0, self.bufs[slot]
        for k, v in sample.items():
            if isinstance(v, np.ndarray):
                dt = torch.from_numpy(np.empty(0, v.dtype)).dtype
                t = buf[off:off + v.nbytes].view(dt).view(v.shape)
                np.copyto(t.numpy(), v)
                out[k] = t
                off += self._span(v)
        return out


class PreparedSamples:
    """Iterates `dataset.prepare(dataset[i], device)` over `indices` in order.  A reader thread reads up to
    `num_workers` images ahead into a ring of pinned buffers (pin_memory=True; _PinnedRing); an exception there is
    raised here."""

    def __init__(self, dataset, indices, device, num_workers=2, pin_memory=True):
        self.dataset, self.indices, self.device = dataset, list(indices), device
        self.depth, self.pin_memory = max(1, int(num_workers)), pin_memory

    def _read(self, indices, ring, q, stop):
        try:
            for i in indices:
                s = self.dataset[i]
                slot = None
                if ring is not None:
                    slot = _get(ring.free, stop)
                    if slot is None:
                        return
                    filled = ring.fill(slot, s)
                    if filled is None:
                        ring.free.put(slot)
                        slot = None
                    else:
                        s = filled
                if not _put(q, stop, ('ok', slot, s)):
                    return
        except BaseException as e:           # handed to the consumer, which raises it
            _put(q, stop, ('error', None, e))

    def __iter__(self):
        if not self.indices:
            return
        first = self.dataset[self.indices[0]]
        ring = None
        if self.pin_memory:
            # slots: queued (depth) + being filled + being copied + one whose copies may still be in flight
            ring = _PinnedRing(first, self.depth + 3)
        q, stop = queue.Queue(maxsize=self.depth), threading.Event()
        th = threading.Thread(target=self._read, args=(self.indices[1:], ring, q, stop), daemon=True)
        pending = []                                            # (event after the copies from a slot, slot)

        def recycle():
            while pending and pending[0][0].query():
                ring.free.put(pending.pop(0)[1])

        try:
            slot, item = None, first
            if ring is not None:
                slot = ring.free.get()
                filled = ring.fill(slot, first)
                if filled is None:
                    ring.free.put(slot)
                    slot = None
                else:
                    item = filled
            th.start()
            for n in range(len(self.indices)):
                if n > 0:
                    got = _get(q, stop, recycle if ring is not None else None)
                    tag, slot, item = got
                    if tag == 'error':
                        raise item
                out = self.dataset.prepare(item, self.device)
                if slot is not None:
                    ev = torch.cuda.Event()
                    ev.record()
                    pending.append((ev, slot))
                    recycle()
                yield out
        finally:
            stop.set()
            if th.is_alive():
                th.join()
            for ev, _ in pending:
                ev.synchronize()


# ------------------------------------------------------------------------- the reference's host preparation (numpy)
def get_boundaries(x, th=1.0):
    """`estimator/utils/image_ops.py:25-36` with dilation=0, as float32 0/1."""
    ey = np.logical_or(np.pad(np.abs(x[1:, :] - x[:-1, :]) > th, ((1, 0), (0, 0))),
                       np.pad(np.abs(x[:-1, :] - x[1:, :]) > th, ((0, 1), (0, 0))))
    ex = np.logical_or(np.pad(np.abs(x[:, 1:] - x[:, :-1]) > th, ((0, 0), (1, 0))),
                       np.pad(np.abs(x[:, :-1] - x[:, 1:]) > th, ((0, 0), (0, 1))))
    return np.logical_or(ey, ex).astype(np.float32)


def host_ground_truth(src, kind, factor=0.0, doffs=0.0):
    """(depth_gt fp32, boundary fp32) of one source map with the reference's numpy arithmetic (u4k_dataset.py:118-119,
    168; general_dataset.py:66-136).  factor / doffs are Python floats, as the reference holds them."""
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        if kind == 'u4k':
            disp = src.astype(np.float32)
            return factor / disp, get_boundaries(disp, th=1)
        if kind == 'mid':
            disp = src.astype(np.float32)
            disp_copy = disp.copy()
            invalid = disp == np.inf
            depth = factor / (disp + doffs)
            depth = depth / 1000
            depth[invalid] = 0
            disp_copy[invalid] = 0
            return depth, get_boundaries(disp_copy, th=1)
        if kind == 'eth3d':
            depth = np.nan_to_num(src, posinf=0., neginf=0., nan=0.).astype(np.float32)
            return depth, get_boundaries(depth, th=1)
        if kind == 'cityscapes':
            d = src.astype(np.float32)
            d[d > 0] = (d[d > 0] - 1) / 256
            depth = np.nan_to_num(factor / d, posinf=0., neginf=0., nan=0.).astype(np.float32)
            return depth, get_boundaries(depth, th=1)
    raise NotImplementedError('ground truth of kind %r' % (kind,))


def host_image(image_u8):
    """u4k_dataset.py:126-129: BGR uint8 -> RGB float32 / 255 (HWC)."""
    return image_u8.astype(np.float32)[:, :, ::-1].copy() / 255.0


def host_prepare(sample, device):
    """The reference's preparation of a raw-frame sample: image and ground truth computed with numpy on the host, then
    copied to the device as fp32 (image_hr, depth_gt, boundary)."""
    if sample['image_resize'] is not None:
        raise NotImplementedError('host_prepare restates the raw-frame path only')
    img = torch.from_numpy(host_image(sample['image'])).permute(2, 0, 1).unsqueeze(0)
    out = dict(image_hr=img.to(device), img_file_basename=sample['img_file_basename'])
    if sample.get('gt') is not None:
        depth, boundary = host_ground_truth(sample['gt'], sample['gt_kind'], sample['factor'], sample['doffs'])
        out['depth_gt'] = torch.from_numpy(depth)[None, None].to(device)
        out['boundary'] = torch.from_numpy(boundary)[None, None].to(device)
    return out
