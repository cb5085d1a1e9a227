"""Post-training calibration of the static FP8 Guided-Fusion U-Net (fusion_precision 'fp8_static').

    python tools/calibrate_fp8.py <config.py> --ckp-path <ckpt> --num-images N --out DIR \
        [--test-type normal] [--cai-mode m1] [--image-raw-shape 2160 3840] [--patch-split-num 4 4] [--cfg-options k=v ...]

Builds the model as tools/test.py does (same config, checkpoint, dataset and tiling arguments), switches it to
'fp8_static', runs PatchFusion.calibrate_fp8 over the first N images of the dataset (read and ingested as the
evaluation reads them) and writes a save_pretrained directory whose config carries fusion_precision 'fp8_static' and the
calibration table `fusion_fp8_amax`.  `tools/test.py <config.py> --ckp-path DIR` then evaluates the calibrated model.
A config that selects dpt_precision 'fp8_static' (`--cfg-options model.config.dpt_precision=fp8_static`) gets the DPT
decoders' table `dpt_fp8_amax` filled, written and printed too.
"""
import argparse
import json
import os
import random
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402


def main(argv=None):
    p = argparse.ArgumentParser(description='Calibrate the static FP8 U-Net of a PatchFusion model')
    p.add_argument('config')
    p.add_argument('--ckp-path', type=str, required=True)
    p.add_argument('--test-type', type=str, default='normal')
    p.add_argument('--cai-mode', type=str, default='m1')
    p.add_argument('--process-num', type=int, default=2)
    p.add_argument('--image-raw-shape', nargs='+', default=[2160, 3840])
    p.add_argument('--patch-split-num', nargs='+', default=[4, 4])
    p.add_argument('--cfg-options', nargs='+', default=None)
    p.add_argument('--num-images', type=int, required=True)
    p.add_argument('--out', type=str, required=True, help='save_pretrained directory to write')
    args = p.parse_args(argv)
    from estimator.datasets import build_dataset
    from patchfusion_b200 import imageio
    from patchfusion_b200.config import load_config, merge_options, parse_options
    from patchfusion_b200.datasets import PreparedSamples
    from patchfusion_b200.evaluate import DATALOADERS, build_model, fix_random_seed
    from patchfusion_b200.model import PatchFusion
    image_raw_shape = [int(v) for v in args.image_raw_shape]
    tile_cfg = {'image_raw_shape': image_raw_shape, 'patch_split_num': [int(v) for v in args.patch_split_num]}
    cfg = load_config(args.config)
    if args.cfg_options:
        merge_options(cfg, parse_options(args.cfg_options))
    fix_random_seed(cfg.get('seed', 5621))
    device = torch.device('cuda', torch.cuda.current_device())
    src = build_model(cfg, args.ckp_path)
    # the same weights in an 'fp8_static' model (the table starts empty: calibrate_fp8 fills it)
    conf = dict(src.config.to_dict(), fusion_precision='fp8_static')
    conf.pop('fusion_fp8_amax', None)
    dpt = conf.get('dpt_precision', 'bf16') == 'fp8_static'     # the DPT decoders' table too
    if dpt:
        conf.pop('dpt_fp8_amax', None)
    model = PatchFusion(conf)
    model.load_state_dict(src.state_dict(), strict=True)
    del src
    model = model.to(device).eval()
    dataset = build_dataset(cfg[DATALOADERS.get(args.test_type, 'val_dataloader')].dataset)
    dataset.image_resolution = image_raw_shape
    n = min(args.num_images, len(dataset))
    table = None
    for s in PreparedSamples(dataset, range(n), device, num_workers=2):
        img = s['image_hr'].to(device).float() if 'image_hr' in s else \
            imageio.ingest(s['image_u8'], tuple(image_raw_shape), device, bgr=True)
        table = model.calibrate_fp8(model.make_lr(img), img, cai_mode=args.cai_mode, process_num=args.process_num,
                                    tile_cfg=tile_cfg)
    if table is None:
        raise SystemExit('calibrate_fp8: the dataset has no images')
    model.save_pretrained(args.out)
    out = dict(images=n, fusion_fp8_amax=table)
    if dpt:
        out['dpt_fp8_amax'] = dict(model.config['dpt_fp8_amax'])
    print(json.dumps(out, indent=1))
    return table


if __name__ == '__main__':
    random.seed(0)
    main()
