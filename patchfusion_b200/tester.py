"""The caller loop of the hot path (SURVEY.md §8f-1): counterpart of `estimator/tester/tester.py:47-95`.

Per image the reference does: model(mode='infer') -> colorize (host numpy + matplotlib) -> cv2.imwrite colour PNG ->
uint16 PNG (depth * 256) -> compute_metrics (host numpy) - all serial, after a synchronous device->host copy of the
8.3 MP fp32 map.  Here everything up to the PNG encoder runs on the GPU (pf_ingest_u8, the model, pf_colorize_u8,
pf_depth_to_u16, pf_depth_metrics); results are copied into pinned double buffers on a side stream and handed to a
host thread that encodes the PNGs while the next image is being computed."""
import os
import queue
import threading

import numpy as np
import torch

from . import imageio, metrics as pf_metrics


class Tester:
    def __init__(self, model, work_dir=None, save=False, gray_scale=False, min_depth=1e-3, max_depth=80.0):
        self.model = model
        self.work_dir, self.save, self.gray_scale = work_dir, save, gray_scale
        self.min_depth, self.max_depth = min_depth, max_depth
        if save:
            os.makedirs(work_dir, exist_ok=True)

    def _writer(self, q):
        import cv2
        while True:
            item = q.get()
            if item is None:
                return
            ev, name, color, raw = item
            ev.synchronize()                                   # the D2H copies of this slot have landed
            cv2.imwrite(os.path.join(self.work_dir, '%s.png' % name), color.numpy())
            cv2.imwrite(os.path.join(self.work_dir, '%s_uint16.png' % name), raw.numpy())
            q.task_done()

    @staticmethod
    def _groups(samples, batch_size):
        """consecutive samples in lists of batch_size (the last one may be shorter), in input order"""
        group = []
        for s in samples:
            group.append(s)
            if len(group) == batch_size:
                yield group
                group = []
        if group:
            yield group

    @torch.no_grad()
    def run(self, samples, cai_mode='m1', process_num=4, image_raw_shape=(2160, 3840), patch_split_num=(4, 4),
            batch_size=1):
        """samples: iterable of dicts {'img_file_basename': str, 'image_u8': HxWx3 uint8 BGR (cv2.imread) OR
        'image_hr': (1,3,H,W) fp32 in [0,1], optional 'depth_gt' (1,1,h,w), optional 'boundary', optional 'tile_cfg'
        ({'image_raw_shape', 'patch_split_num'}) and 'cai_mode'}.  A sample without its own tile_cfg / cai_mode uses
        the run's (image_raw_shape, patch_split_num, cai_mode).
        batch_size > 1: consecutive samples go through the model together (one batched forward; samples of different
        geometry or mode form a mixed batch); outputs, files and metrics are those of batch_size 1, in input order.
        Returns the list of per-image metric dicts (empty when no ground truth is given)."""
        model = self.model
        dev = next(model.parameters()).device
        default_cfg = {'image_raw_shape': list(image_raw_shape), 'patch_split_num': list(patch_split_num)}
        results = []
        copy_stream = torch.cuda.Stream(device=dev)
        slots, q, th = [None, None], None, None
        if self.save:
            q = queue.Queue(maxsize=2)
            th = threading.Thread(target=self._writer, args=(q,), daemon=True)
            th.start()
        i = 0
        for group in self._groups(samples, max(1, int(batch_size))):
            cfgs = [s.get('tile_cfg', default_cfg) for s in group]
            modes = [s.get('cai_mode', cai_mode) for s in group]
            images = []
            for s, cfg in zip(group, cfgs):
                if 'image_hr' in s:
                    images.append(s['image_hr'].to(dev, non_blocking=True).float())
                else:
                    images.append(imageio.ingest(s['image_u8'], tuple(cfg['image_raw_shape']), dev, bgr=True))
            keys = {(tuple(c['image_raw_shape']), tuple(c['patch_split_num']), m) for c, m in zip(cfgs, modes)}
            if len(keys) == 1:
                image = images[0] if len(images) == 1 else torch.cat(images)
                lr = model.make_lr(image)
                results_b, _ = model(mode='infer', cai_mode=modes[0], process_num=process_num, tile_cfg=cfgs[0],
                                     image_lr=lr, image_hr=image)
                results_b = [results_b[j:j + 1] for j in range(len(group))]
            else:
                results_b, _ = model(mode='infer', cai_mode=modes, process_num=process_num, tile_cfg=cfgs,
                                     image_lr=model.make_lr(images), image_hr=images)
            for j, s in enumerate(group):
                result = results_b[j]
                self._emit(s, i, result, slots, q, copy_stream, dev, results)
                i += 1
        if self.save:
            q.join()
            q.put(None)
            th.join()
        return results

    def _emit(self, s, i, result, slots, q, copy_stream, dev, results):
        """Outputs of sample number i: colour and uint16 PNGs through the writer thread, metrics."""
        if self.save:
            color = imageio.colorize(result, cmap='gray_r' if self.gray_scale else 'magma_r', bgr=True)
            raw = imageio.depth_to_u16(result)              # tester.py:75: (result * 256).astype('uint16')
            k = i % 2
            if slots[k] is None or slots[k][0].shape != color.shape:
                slots[k] = (torch.empty(color.shape, dtype=torch.uint8).pin_memory(),
                            torch.empty(raw.shape, dtype=torch.uint16).pin_memory())
            q.join() if i >= 2 and q.unfinished_tasks >= 2 else None
            ev = torch.cuda.Event()
            copy_stream.wait_stream(torch.cuda.current_stream(dev))
            with torch.cuda.stream(copy_stream):
                slots[k][0].copy_(color, non_blocking=True)
                slots[k][1].copy_(raw, non_blocking=True)
                ev.record(copy_stream)
            color.record_stream(copy_stream)
            raw.record_stream(copy_stream)
            q.put((ev, s['img_file_basename'], slots[k][0], slots[k][1]))
        if s.get('depth_gt') is not None:
            results.append(pf_metrics.compute_metrics(
                s['depth_gt'].to(dev), result, disp_gt_edges=s.get('boundary'), min_depth_eval=self.min_depth,
                max_depth_eval=self.max_depth))

    @staticmethod
    def evaluate(results):
        """u4k_dataset.py:188-210: nanmean of every metric over the images."""
        keys = list(results[0].keys()) if results else []
        return {k: float(np.nanmean([r[k] for r in results])) for k in keys}
