"""DVT stage 2 (training the generalizable denoiser) on H100 -- drop-in for the reference's main_denoiser.py.

Same flags (reference main_denoiser.py:25-78 incl. `--auto_stride` and the 518 -> 512 rule for stride 16 / 8), same model
(`dvt.models.Denoiser(vit=None, num_blocks)`, :129-135), same objective (MSE + 1 - mean cosine, :214-217), AdamW with
betas (0.9, 0.999) and weight decay on every parameter (:176-180), sqrt-scaled learning rate and the 15 %-warm-up cosine
schedule (:174,181-188), same checkpoint layout `{"denoiser", "optimizer", "step"}` + `latest.pth` symlink (:239-264).

What runs where: forward and backward of the transformer block, the loss with its gradient and the AdamW update are
hand-written sm_90a kernels (dvt/train_ops.py, dvt/optim.py); data parallelism is ONE NCCL all-reduce of the flat
gradient buffer per step (the reference wraps the model in DistributedDataParallel, :137-140).  Launch with torchrun
(RANK / WORLD_SIZE / LOCAL_RANK from the environment), one process per GPU.

H100 extension: `--collated <file.pt>` trains straight from the tensors stage 1 gathered with its all-gather
(`main_img_denoising.py --collate_out`), held in HBM, instead of re-reading the `.npy` store.
The PCA visualisation (reference :266-275) is outside the hot path and not produced."""
import argparse
import datetime
import math
import os
import re
import sys
import time

import numpy as np
import torch
import torchvision.transforms as transforms
from PIL import Image

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "denoising-vit_b200"))

import dvt.dataset as dataset  # noqa: E402
import dvt.models as DVT  # noqa: E402
from dvt import train_ops  # noqa: E402
from dvt.optim import FusedAdamW  # noqa: E402
from dvt.utils import misc  # noqa: E402


def get_args(argv=None):
    parser = argparse.ArgumentParser("Train generalizable denoiser", add_help=False)
    # model
    parser.add_argument("--model", type=str, default="vit_base_patch14_dinov2.lvd142m", choices=DVT.MODEL_LIST)
    parser.add_argument("--num_blocks", type=int, default=1)
    # data
    parser.add_argument("--data_root", type=str, default="data/imagenet")
    parser.add_argument("--feat_root", type=str, default=None)
    parser.add_argument("--data_list_path", type=str, default=None)
    parser.add_argument("--input_size", type=int, default=518, nargs="+")
    parser.add_argument("--auto_stride", action="store_true", help="set stride size = patch size.")
    parser.add_argument("--stride_size", type=int, default=14, help="Stride size for the model.")
    parser.add_argument("--num_workers", default=8, type=int)
    # training
    parser.add_argument("--batch_size", default=32, type=int, help="Batch size per GPU")
    parser.add_argument("--num_vis_samples", default=8, type=int)
    parser.add_argument("--num_iterations", default=40_000, type=int)
    # Optimizer parameters
    parser.add_argument("--weight_decay", type=float, default=1e-5)
    parser.add_argument("--blr", type=float, default=2.0e-04, help="abs_lr = blr * total_bs / 256")
    parser.add_argument("--min_lr", type=float, default=1.0e-06, help="for cosine scheduler")
    parser.add_argument("--warmup_iters", type=int, default=50_000, help="iterations to warmup LR")
    # logging
    parser.add_argument("--output_root", default="./work_dirs/", type=str)
    parser.add_argument("--save_freq", default=5000, type=int)
    parser.add_argument("--vis_freq", default=5000, type=int)
    parser.add_argument("--project", default="denosing-vit", type=str)
    parser.add_argument("--run_name", default="debug", type=str)
    parser.add_argument("--seed", default=42, type=int)
    parser.add_argument("--world_size", default=1, type=int, help="number of distributed processes")
    parser.add_argument("--local_rank", "--local-rank", default=-1, type=int)
    parser.add_argument("--dist_on_itp", action="store_true")
    parser.add_argument("--dist_url", default="env://")
    parser.add_argument("--distributed", action="store_true")
    parser.add_argument("--device", default="cuda", help="device to use for training / testing")
    # H100 extensions (not reference flags)
    parser.add_argument("--collated", type=str, default=None,
                        help="train from the in-memory stacks written by main_img_denoising.py --collate_out")
    parser.add_argument("--resume", type=str, default=None, help="checkpoint to continue from (e.g. .../latest.pth)")
    parser.add_argument("--log_freq", default=50, type=int)
    parser.add_argument("--deterministic", action="store_true",
                        help="torch.use_deterministic_algorithms(True): fixed-order backward kernels, so that a rerun from "
                             "the same seed on the same GPU model gives bit-identical weights and losses")
    args = parser.parse_args(argv)

    if isinstance(args.input_size, int):
        args.input_size = (args.input_size, args.input_size)
    elif len(args.input_size) == 1:
        args.input_size = (args.input_size[0], args.input_size[0])
    args.input_size = list(args.input_size)
    if args.auto_stride:
        args.stride_size = int(re.search(r"patch(14|16)", args.model).group(1))
        print(f"Auto set stride to {args.stride_size}")
    if (args.stride_size == 16 or args.stride_size == 8) and args.input_size[0] == 518:
        args.input_size = [512, 512]
        print(f"Set input size to {args.input_size}")
    assert args.input_size[0] % args.stride_size == 0, "height must be divisible by stride_size"
    assert args.input_size[1] % args.stride_size == 0, "width must be divisible by stride_size"
    return args


def save_checkpoint(log_dir: str, model, optimizer, step: int):
    """main_denoiser.py:239-264: everything but the frozen backbone, torch.optim-style optimiser state, `latest.pth`."""
    state = {k: v for k, v in model.state_dict().items() if "vit." not in k}
    path = f"{log_dir}/checkpoints/ckpt_{step:06d}.pth"
    torch.save({"denoiser": state, "optimizer": optimizer.state_dict(), "step": step}, path)
    latest = f"{log_dir}/checkpoints/latest.pth"
    try:
        os.remove(latest)
    except FileNotFoundError:
        pass
    os.symlink(os.path.abspath(path), latest)
    print(f"Saved checkpoint to {path}; {latest} -> {path}")
    return path


def main(args):
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    assert torch.cuda.is_available(), "the H100 stage-2 trainer needs a CUDA device (no CPU fallback)"
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=device)
    log_dir = os.path.join(args.output_root, args.project, args.run_name)
    if rank == 0:
        os.makedirs(f"{log_dir}/checkpoints", exist_ok=True)
        print("\n".join(f"{k}: {v}" for k, v in sorted(vars(args).items())))
    misc.fix_random_seeds(args.seed)
    if args.deterministic:
        torch.use_deterministic_algorithms(True)

    # the backbone is needed for its geometry only (the reference builds it, reads patch size / width and deletes it)
    m = re.search(r"patch(\d+)", args.model)
    patch = int(m.group(1))
    from dvt.models import vit_wrapper as VW
    if args.model not in VW.ARCHS:
        raise NotImplementedError(f"{args.model}: architecture outside the supported ViT family")
    args.feat_dim = VW.ARCHS[args.model]["embed"]
    pos_h = (args.input_size[0] - patch) // args.stride_size + 1
    pos_w = (args.input_size[1] - patch) // args.stride_size + 1
    args.noise_map_height, args.noise_map_width = pos_h, pos_w

    model = DVT.Denoiser(noise_map_height=pos_h, noise_map_width=pos_w, feat_dim=args.feat_dim, vit=None,
                         num_blocks=args.num_blocks).to(device)
    if world > 1:  # every rank starts from rank 0's initialisation (what DistributedDataParallel does at construction)
        import torch.distributed as dist
        for p in model.parameters():
            dist.broadcast(p.data, 0)
    if rank == 0:
        print(f"Model = {model}")

    if args.collated is not None:
        packed = torch.load(args.collated, map_location="cpu")
        train_dataset = dataset.InMemoryPairs(packed["raw_feats"].to(device), packed["denoised_feats"].to(device))
    else:
        arch = VW.ARCHS[args.model]
        train_dataset = dataset.FeatureStoreDataset(
            data_root=args.data_root, feat_root=args.feat_root, data_list=args.data_list_path,
            transform=transforms.Compose([transforms.Resize(args.input_size, interpolation=Image.BICUBIC, antialias=True),
                                          transforms.ToTensor(), transforms.Normalize(arch["mean"], arch["std"])]))
    print(f"Dataset size: {len(train_dataset)}")
    sampler = (dataset.DistributedInfiniteSampler(train_dataset, num_replicas=world, rank=rank) if world > 1
               else dataset.InfiniteSampler(train_dataset))
    in_memory = isinstance(train_dataset, dataset.InMemoryPairs)
    data_loader = torch.utils.data.DataLoader(train_dataset, batch_size=args.batch_size, sampler=sampler,
                                              num_workers=0 if in_memory else args.num_workers,
                                              pin_memory=not in_memory, drop_last=False)

    args.lr = args.blr * math.sqrt(args.batch_size * world / 256)
    print(f"sqrt scaling learning rate; blr: {args.blr}, actual lr: {args.lr}")
    optimizer = FusedAdamW(model.parameters(), betas=(0.9, 0.999), weight_decay=args.weight_decay)
    sched = dict(base_value=args.lr, final_value=args.min_lr, total_iters=args.num_iterations,
                 warmup_iters=int(args.num_iterations * 0.15), start_warmup_value=0)
    start_step = 0
    if args.resume:
        ck = torch.load(args.resume, map_location=device)
        model.load_state_dict(ck["denoiser"], strict=False)
        optimizer.load_state_dict(ck["optimizer"])
        start_step = int(ck["step"]) + 1
        print(f"Resumed from {args.resume} at step {start_step}")

    model.train()
    end = start = time.time()
    window = []
    it = iter(data_loader)
    for step in range(start_step, args.num_iterations):
        data_dict = next(it)
        feats = data_dict["original_feats"].to(device, non_blocking=True)
        target = data_dict["denoised_feats"].to(device, non_blocking=True)
        data_time = time.time() - end
        lr = misc.cosine_schedule(step, **sched)
        misc.apply_optim_scheduler(optimizer, lr)
        pred = model(feats)
        loss, l2_loss, cos_loss = train_ops.denoise_loss(pred, target)
        optimizer.zero_grad()
        loss.backward()
        optimizer.sync_grads(world)
        optimizer.step()
        window.append(torch.stack([loss.detach(), l2_loss.detach(), cos_loss.detach()]))
        if step % args.log_freq == 0 or step == args.num_iterations - 1:
            vals = torch.stack(window).mean(0).tolist()       # the only host synchronisation of the loop
            window = []
            if not all(math.isfinite(v) for v in vals):
                print(f"Loss is {vals[0]}, stopping training")
                sys.exit(1)
            iter_time = (time.time() - end)
            eta = (time.time() - start) / max(1, step - start_step + 1) * (args.num_iterations - step - 1)
            if rank == 0:
                print(f"Train [{step:>6}/{args.num_iterations}] eta: {datetime.timedelta(seconds=int(eta))} "
                      f"loss: {vals[0]:.4f} l2_loss: {vals[1]:.4f} cosine_similarity_loss: {vals[2]:.4f} "
                      f"data_time: {data_time:.4f} iter_time: {iter_time:.4f} lr: {lr:.6g}", flush=True)
        if rank == 0 and (step % args.save_freq == 0 or step == args.num_iterations - 1):
            save_checkpoint(log_dir, model, optimizer, step)
        end = time.time()
    torch.cuda.synchronize()
    if rank == 0:
        print(f"Total time: {datetime.timedelta(seconds=int(time.time() - start))}")
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main(get_args())
