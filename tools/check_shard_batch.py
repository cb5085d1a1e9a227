"""torchrun --nproc-per-node N tools/check_shard_batch.py : a batch of 3 images, tile-sharded over N GPUs (coarse
stages spread over the owner ranks, one all-gather of their packs, one all-gather of the prediction blocks) == the
same batch on one GPU, bit for bit, in both coarse modes and m1 / m2 / r4."""
import os, sys, random
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist
from patchfusion_b200.configs import depth_anything_patchfusion
from patchfusion_b200.model import PatchFusion
from patchfusion_b200.params import synthetic_state_dict

rank, world, local = int(os.environ['RANK']), int(os.environ['WORLD_SIZE']), int(os.environ['LOCAL_RANK'])
dev = torch.device('cuda', local)
torch.cuda.set_device(dev)
dist.init_process_group('nccl', device_id=dev)
cfg = depth_anything_patchfusion('vits', image_raw_shape=(1080, 1920), patch_split_num=(2, 2))
model = PatchFusion(cfg)
model.load_state_dict(synthetic_state_dict(cfg, seed=0))
model = model.to(dev).eval()
img = torch.rand(3, 3, 1080, 1920, generator=torch.Generator().manual_seed(0)).to(dev)
lr = model.make_lr(img)
ok = True
for how in ('owner', 'replicate'):
    model.shard_coarse = how
    for mode in ('m1', 'm2', 'r4'):
        random.seed(0)
        ref, _ = model(mode='infer', image_lr=lr, image_hr=img, cai_mode=mode, process_num=2)
        ref = ref.clone()
        for rep in range(2):             # second pass replays the captured graphs
            random.seed(0)
            y, _ = model(mode='infer', image_lr=lr, image_hr=img, cai_mode=mode, process_num=2, shard=(rank, world))
            err = (y - ref).abs().max().item()
            t = torch.tensor([err], device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            if rank == 0:
                print('B=3 %s %s pass %d: world %d  max|sharded - single| = %.3e (range %.3f..%.3f)'
                      % (how, mode, rep, world, t.item(), ref.min().item(), ref.max().item()), flush=True)
            ok = ok and t.item() == 0.0
dist.barrier()
dist.destroy_process_group()
sys.exit(0 if ok else 1)
