"""python tools/check_eval_shard.py [--out DIR] : image-sharded evaluation on every visible GPU against one GPU.

Writes a synthetic U4K case (5 frames, vits synthetic weights) and runs tools/test.py's logic under torchrun on all
visible GPUs (--launcher pytorch) for m1 and r4.  Every rank seeds itself with the config seed, so random tiles restart
per rank, as in the reference's distributed run.  The W-rank metrics.json and PNGs are therefore compared, byte for
byte, with `evaluate.shard_reference` on one GPU: each rank's shard range(r, n, W) in order, reseeded first.  For m1,
which draws nothing at random, they must also equal the plain one-GPU run.  Exit status 0 when all are equal."""
import argparse
import filecmp
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def cli_args(conf, ckpt, mode, work_dir):
    return [conf, '--ckp-path', ckpt, '--cai-mode', mode, '--save', '--gray-scale', '--work-dir', work_dir,
            '--image-raw-shape', '2160', '3840', '--patch-split-num', '2', '2']


def same_pngs(a, b):
    fa = sorted(f for f in os.listdir(a) if f.endswith('.png'))
    return len(fa), fa == sorted(f for f in os.listdir(b) if f.endswith('.png')) and all(
        filecmp.cmp(os.path.join(a, f), os.path.join(b, f), shallow=False) for f in fa)


def main():
    import torch
    from estimator.datasets import build_dataset
    from patchfusion_b200 import eval_tree
    from patchfusion_b200.config import load_config
    from patchfusion_b200.evaluate import build_model, main as evaluate, shard_reference
    from patchfusion_b200.tester import Tester
    p = argparse.ArgumentParser()
    p.add_argument('--out', default=None)
    args = p.parse_args()
    world = torch.cuda.device_count()
    dev = torch.device('cuda', 0)
    tmp = tempfile.mkdtemp(prefix='pf_eval_shard_')
    conf, ckpt, _ = eval_tree.write_u4k_case(tmp, n_frames=5)
    cfg = load_config(conf)
    ds = build_dataset(cfg.val_dataloader.dataset)
    model = build_model(cfg, ckpt).to(dev).eval()
    ok, report = True, {'gpus': world, 'card': torch.cuda.get_device_name(0)}
    for mode in ('m1', 'r4'):
        ref, many = os.path.join(tmp, 'shard_ref_' + mode), os.path.join(tmp, 'many_' + mode)
        tester = Tester(model, work_dir=ref, save=True, gray_scale=True, min_depth=ds.min_depth,
                        max_depth=ds.max_depth)
        want = json.loads(json.dumps(dict(ds.evaluate(shard_reference(
            tester, ds, dev, world, cfg.get('seed', 5621), cai_mode=mode, process_num=2, image_raw_shape=(2160, 3840),
            patch_split_num=(2, 2))))))
        subprocess.check_call(['torchrun', '--standalone', '--nproc-per-node', str(world),
                               os.path.join(ROOT, 'tools', 'test.py')] + cli_args(conf, ckpt, mode, many) +
                              ['--launcher', 'pytorch'], cwd=ROOT)
        got = json.load(open(os.path.join(many, 'metrics.json')))
        n_png, files = same_pngs(ref, many)
        rec = dict(metrics_equal=got == want, files_equal=files, n_png=n_png, metrics=got)
        good = got == want and files and n_png == 2 * len(ds)
        if mode == 'm1':
            one = os.path.join(tmp, 'one_' + mode)
            m_one = evaluate(cli_args(conf, ckpt, mode, one))
            n1, files1 = same_pngs(one, many)
            rec.update(one_gpu_metrics_equal=json.loads(json.dumps(m_one)) == got, one_gpu_files_equal=files1)
            good = good and rec['one_gpu_metrics_equal'] and files1 and n1 == n_png
        report[mode] = rec
        ok = ok and good
        print(mode, rec, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        json.dump(report, open(os.path.join(args.out, 'check_eval_shard.json'), 'w'), indent=1)
    print('check_eval_shard: %s on %d GPUs' % ('OK' if ok else 'MISMATCH', world))
    sys.exit(0 if ok else 1)


if __name__ == '__main__':
    main()
