"""Dataset evaluation: the logic of `tools/test.py` (reference `tools/test.py:18-251`), callable in-process.

    python tools/test.py <config.py> --ckp-path <ckpt> --cai-mode <m1|m2|rN> --test-type <normal|test_in|test_out|general>
        [--save] [--gray-scale] --work-dir <dir> --image-raw-shape H W --patch-split-num h w [--cfg-options k=v ...]
        [--launcher pytorch]

Images go through `PreparedSamples` (raw sources read on a reader thread, prepared on the GPU) into `Tester.run`.
Under `--launcher pytorch` (torchrun environment, NCCL) images are sharded like the reference's
`DistributedSampler(shuffle=False)` + `collect_results_gpu`: rank r takes indices r, r + W, ... of the list padded to a
multiple of W, except that the padded duplicates are not computed (the reference computes and then drops them).  Each
rank seeds with the config seed and runs its images in order, so rN outputs equal the reference's distributed run.
Per-image metrics travel as fixed-size fp64 rows in one all-gather; interleaving them by rank and truncating to N gives
the single-process list, which rank 0 evaluates."""
import argparse
import json
import logging
import os
import os.path as osp
import random
import sys
import time

import numpy as np
import torch

from .config import load_config, merge_options, parse_options
from .datasets import METRIC_KEYS, PreparedSamples

HUB_IDS = ('Zhyever/patchfusion_depth_anything_vits14', 'Zhyever/patchfusion_depth_anything_vitb14',
           'Zhyever/patchfusion_depth_anything_vitl14', 'Zhyever/patchfusion_zoedepth')
DATALOADERS = {'normal': 'val_dataloader', 'test_in': 'test_in_dataloader', 'test_out': 'test_out_dataloader',
               'general': 'general_dataloader'}
ROW = 2 + len(METRIC_KEYS)          # [computed, has_see, a1 ... sq_rel, see]


def parse_args(argv=None):
    p = argparse.ArgumentParser(description='Evaluate a PatchFusion model on a dataset')
    p.add_argument('config', help='config file path')
    p.add_argument('--work-dir', default=None, help='the dir to save logs and predictions')
    p.add_argument('--test-type', type=str, default='normal', help='normal, test_in, test_out or general')
    p.add_argument('--ckp-path', type=str, help='a .pth checkpoint, a hub id or a save_pretrained directory')
    p.add_argument('--amp', action='store_true', default=False, help='accepted for compatibility; inference is fp32')
    p.add_argument('--save', action='store_true', default=False, help='save colored prediction & depth predictions')
    p.add_argument('--cai-mode', type=str, default='m1', help='m1, m2, or rN')
    p.add_argument('--process-num', type=int, default=2, help='tiles per micro-batch')
    p.add_argument('--tag', type=str, default='', help='infer_infos')
    p.add_argument('--gray-scale', action='store_true', default=False, help='use gray-scale color map')
    p.add_argument('--image-raw-shape', nargs='+', default=[2160, 3840])
    p.add_argument('--patch-split-num', nargs='+', default=[4, 4])
    p.add_argument('--cfg-options', nargs='+', default=None, help='key=value overrides of the config (mmengine syntax)')
    p.add_argument('--launcher', choices=['none', 'pytorch', 'slurm', 'mpi'], default='none', help='job launcher')
    p.add_argument('--local_rank', '--local-rank', type=int, default=0)
    args = p.parse_args(argv)
    if 'LOCAL_RANK' not in os.environ:
        os.environ['LOCAL_RANK'] = str(args.local_rank)
    return args


def fix_random_seed(seed):
    """`estimator/utils/misc.py:16-26`: every generator the tiled forward can draw from."""
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    torch.cuda.manual_seed_all(seed)
    torch.backends.cudnn.deterministic = True
    torch.backends.cudnn.benchmark = True


def shard_indices(n, rank, world):
    """DistributedSampler(shuffle=False) indices of `rank` that are real images: r, r + W, ... < n.  The padding the
    sampler appends (indices 0, 1, ... again, to make n a multiple of W) is left out."""
    return list(range(rank, n, world))


def metric_rows(results, n, world):
    """This rank's per-image metric dicts as fixed-size fp64 rows [ceil(n / W), ROW]; rows past the rank's images are
    zero (not computed)."""
    rows = np.zeros((max(-(-n // world), 1), ROW), dtype=np.float64)
    for j, r in enumerate(results):
        rows[j, 0] = 1.0
        rows[j, 1] = 1.0 if 'see' in r else 0.0
        rows[j, 2:2 + len(r)] = [float(r[k]) for k in METRIC_KEYS[:len(r)]]
    return rows


def interleave_rows(gathered, n):
    """gathered [W, per, ROW] -> the per-image metric dicts of images 0 .. n-1 (image i = row i // W of rank i % W);
    empty when the dataset has no ground truth (no rank computed metrics)."""
    world = gathered.shape[0]
    if not gathered[..., 0].any():
        return []
    out = []
    for i in range(n):
        row = gathered[i % world, i // world]
        assert row[0] == 1.0, 'image %d was not computed' % i
        keys = METRIC_KEYS if row[1] else METRIC_KEYS[:-1]
        out.append({k: float(v) for k, v in zip(keys, row[2:2 + len(keys)])})
    return out


def gather_metrics(results, n, world, device, group=None):
    """One all-gather of every rank's metric rows -> the single-process metric list (on every rank)."""
    import torch.distributed as dist
    rows = torch.from_numpy(metric_rows(results, n, world))
    if dist.get_backend(group) == 'nccl':
        rows = rows.to(device)
    full = torch.empty((world,) + tuple(rows.shape), dtype=rows.dtype, device=rows.device)
    if dist.get_backend(group) == 'nccl':
        dist.all_gather_into_tensor(full, rows, group=group)
    else:
        dist.all_gather(list(full.unbind(0)), rows, group=group)
    return interleave_rows(full.cpu().numpy(), n)


def run_images(tester, dataset, device, rank, world, num_workers=2, **run_kwargs):
    """Evaluate this rank's share of `dataset` with `tester.run` and return the metrics of all images (every rank)."""
    n = len(dataset)
    samples = PreparedSamples(dataset, shard_indices(n, rank, world), device, num_workers=num_workers,
                              pin_memory=torch.cuda.is_available())
    results = tester.run(samples, **run_kwargs)
    if world == 1:
        return results
    return gather_metrics(results, n, world, device)        # every rank joins, also one with no image


def shard_reference(tester, dataset, device, world, seed, num_workers=2, **run_kwargs):
    """What a W-rank run computes, on one device: the shards range(r, n, W) one after another, each in order and
    reseeded with `seed` first (every rank seeds itself, so random tiles (rN) restart per rank), their metrics
    interleaved as the all-gather does.  Equal to the single-process list for deterministic modes only."""
    n = len(dataset)
    per_rank = []
    for r in range(world):
        fix_random_seed(seed)
        samples = PreparedSamples(dataset, shard_indices(n, r, world), device, num_workers=num_workers,
                                  pin_memory=torch.cuda.is_available())
        per_rank.append(tester.run(samples, **run_kwargs))
    return interleave_rows(np.stack([metric_rows(res, n, world) for res in per_rank]), n)


def build_model(cfg, ckp_path):
    """tools/test.py:201-215: a .pth checkpoint goes through build_model(cfg.model) + load_dict; anything else is a
    hub id or a local save_pretrained directory."""
    from patchfusion_b200.model import PatchFusion
    if '.pth' in ckp_path:
        from estimator.models import build_model as _build
        model = _build(cfg.model.to_dict() if hasattr(cfg.model, 'to_dict') else dict(cfg.model))
        logging.getLogger('patchfusion').info('Checkpoint Path: %s. Loading from a local file', ckp_path)
        model.load_dict(torch.load(ckp_path, map_location='cpu')['model_state_dict'])
        return model
    if not osp.isdir(ckp_path) and ckp_path not in HUB_IDS:
        raise ValueError('Invalid model name %r (a .pth checkpoint, a save_pretrained directory or one of %s)' %
                         (ckp_path, ', '.join(HUB_IDS)))
    logging.getLogger('patchfusion').info('Checkpoint Path: %s. Loading from the huggingface repo', ckp_path)
    return PatchFusion.from_pretrained(ckp_path)


def _logger(log_file):
    log = logging.getLogger('patchfusion')
    log.setLevel(logging.INFO)
    for h in list(log.handlers):
        log.removeHandler(h)
        h.close()
    fmt = logging.Formatter('%(asctime)s - %(name)s - %(levelname)s - %(message)s')
    for h in (logging.FileHandler(log_file, mode='a'), logging.StreamHandler(sys.stdout)):
        h.setFormatter(fmt)
        log.addHandler(h)
    log.propagate = False
    return log


def summary_table(ret):
    names = list(ret)
    vals = ['%s' % np.round(ret[k], 7) for k in names]
    widths = [max(len(a), len(b)) + 2 for a, b in zip(names, vals)]
    line = '+' + '+'.join('-' * w for w in widths) + '+'
    return '\n'.join([line, '|' + '|'.join(a.center(w) for a, w in zip(names, widths)) + '|', line,
                      '|' + '|'.join(b.center(w) for b, w in zip(vals, widths)) + '|', line])


def main(argv=None):
    """Run one evaluation; returns the metric dict on rank 0 (None on other ranks or without ground truth)."""
    args = parse_args(argv)
    image_raw_shape = [int(v) for v in args.image_raw_shape]
    patch_split_num = [int(v) for v in args.patch_split_num]
    cfg = load_config(args.config)
    cfg.launcher = args.launcher
    if args.cfg_options:
        merge_options(cfg, parse_options(args.cfg_options))
    # work_dir: CLI > config > next to a .pth checkpoint / work_dir/<hub repo name>
    if args.work_dir is not None:
        cfg.work_dir = args.work_dir
    elif cfg.get('work_dir', None) is None:
        cfg.work_dir = (osp.dirname(args.ckp_path) if '.pth' in args.ckp_path
                        else osp.join('work_dir', args.ckp_path.split('/')[1]))
    os.makedirs(cfg.work_dir, exist_ok=True)
    cfg.ckp_path = args.ckp_path
    seed = cfg.get('seed', 5621)
    fix_random_seed(seed)

    if args.test_type == 'consistency':
        raise NotImplementedError('--test-type consistency: the reference calls a Tester method that does not exist '
                                  '(tools/test.py:249); it is not built here')
    if cfg.launcher == 'none':
        rank, world = 0, 1
        device = torch.device('cuda', torch.cuda.current_device())
        timestamp = time.strftime('%Y%m%d_%H%M%S', time.localtime())
    elif cfg.launcher == 'pytorch':
        import torch.distributed as dist
        local = int(os.environ['LOCAL_RANK'])
        torch.cuda.set_device(local)
        device = torch.device('cuda', local)
        own_group = not dist.is_initialized()
        if own_group:
            dist.init_process_group('nccl', device_id=device)
        rank, world = dist.get_rank(), dist.get_world_size()
        stamp = torch.tensor([time.time()], dtype=torch.float64, device=device)
        dist.broadcast(stamp, 0)                       # one log name for every rank (mmengine setup_env)
        timestamp = time.strftime('%Y%m%d_%H%M%S', time.localtime(stamp.item()))
    else:
        raise NotImplementedError('--launcher %s: only none and pytorch (torchrun) are built' % cfg.launcher)

    from estimator.datasets import build_dataset
    loader_cfg = cfg[DATALOADERS.get(args.test_type, 'val_dataloader')]
    dataset = build_dataset(loader_cfg.dataset)
    dataset.image_resolution = image_raw_shape

    exp_cfg_filename = args.config.split('/')[-1].split('.')[0]
    ckp_name = args.ckp_path.replace('/', '_').replace('.pth', '')
    log_filename = 'eval_{}_{}_{}_{}_{}.log'.format(exp_cfg_filename, args.tag, ckp_name, dataset.dataset_name,
                                                    timestamp)
    log = _logger(osp.join(cfg.work_dir, log_filename)) if rank == 0 else logging.getLogger('patchfusion.rank')

    model = build_model(cfg, args.ckp_path).to(device).eval()

    from .tester import Tester
    tester = Tester(model, work_dir=cfg.work_dir, save=args.save, gray_scale=args.gray_scale,
                    min_depth=dataset.min_depth, max_depth=dataset.max_depth)
    results = run_images(tester, dataset, device, rank, world, num_workers=loader_cfg.get('num_workers', 2),
                         cai_mode=args.cai_mode, process_num=args.process_num, image_raw_shape=image_raw_shape,
                         patch_split_num=patch_split_num)
    ret = None
    if results and rank == 0:
        ret = dataset.evaluate(results)
        log.info('Evaluation Summary: \n' + summary_table(ret))
        with open(osp.join(cfg.work_dir, 'metrics.json'), 'w') as f:
            json.dump(dict(ret), f, indent=1)
    if cfg.launcher == 'pytorch':
        import torch.distributed as dist
        dist.barrier()
        if own_group:
            dist.destroy_process_group()
    return ret
