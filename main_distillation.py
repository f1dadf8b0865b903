"""DVT stage 3 (distilling the denoiser into the backbone) on H100 -- drop-in for the reference's main_distillation.py.

Same flags (reference main_distillation.py:26-80, incl. `--auto_stride`, the 518 -> 512 rule for stride 16 / 8 and the
`--warmup_iters` flag that the reference parses but does not use), same models: the student is
`PretrainedViTWrapper(--model, stride)` trained as a whole, the teacher is the frozen `Denoiser(vit=PretrainedViTWrapper(...),
num_blocks)` with the stage-2 checkpoint `torch.load(--denoiser_ckpt)["denoiser"]` loaded with strict=False (:120-141).
Same objective (MSE + 1 - mean cosine between the student's last-layer features and the teacher's denoised features,
:233-238), same data (`ImageFolder` + bicubic Resize + RandomHorizontalFlip + Normalize, infinite sampler, :157-186), the
number of iterations `steps_per_epoch * num_epochs` when unset, sqrt-scaled learning rate and the 15 %-warm-up cosine
schedule (:187-205), AdamW with betas (0.9, 0.999) over every backbone parameter, and the checkpoint layout
`{"model": wrapper.state_dict(), "optimizer", "step"}` (keys `model.<timm key>`) + `latest.pth` symlink (:256-273).

What runs where: the teacher forward, the student forward and backward (patch embedding, LayerScale blocks, final norm),
the loss with its gradient and the AdamW update are hand-written sm_90a kernels (dvt/models, dvt/train_ops.py,
dvt/optim.py); data parallelism is ONE NCCL all-reduce of the flat gradient buffer per step (the reference wraps the model
in DistributedDataParallel, :146-151).  Launch with torchrun (RANK / WORLD_SIZE / LOCAL_RANK from the environment), one
process per GPU.  Images are decoded and resized by CPU DataLoader workers, as in the reference.

Extensions: `--resume <ckpt>` continues a run, `--log_freq` sets how often the losses are read back (the only host
synchronisation of the loop).  The PCA visualisation of the reference (:275-283) is not produced: it needs imageio and
matplotlib, which this build does not ship."""
import argparse
import datetime
import math
import os
import re
import sys
import time

import torch
import torchvision.transforms as transforms
from PIL import Image
from torchvision.datasets import ImageFolder

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
    parser.add_argument("--denoiser_ckpt", type=str, required=True)
    parser.add_argument("--grad_checkpointing", action="store_true")
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
    parser.add_argument("--num_iterations", default=None, type=int)
    parser.add_argument("--num_epochs", default=10, type=int)
    # Optimizer parameters
    parser.add_argument("--weight_decay", type=float, default=1e-5)
    parser.add_argument("--blr", type=float, default=2.0e-04, help="abs_lr = blr * total_bs / 256")
    parser.add_argument("--min_lr", type=float, default=1.0e-06, help="for cosine scheduler")
    parser.add_argument("--warmup_iters", type=int, default=50_000, help="iterations to warmup LR (unused, as in the reference)")
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


def save_checkpoint(log_dir: str, wrapper, optimizer, step: int):
    """main_distillation.py:256-273: the whole student wrapper, torch.optim-style optimiser state, `latest.pth`."""
    path = f"{log_dir}/checkpoints/ckpt_{step:06d}.pth"
    torch.save({"model": wrapper.state_dict(), "optimizer": optimizer.state_dict(), "step": step}, path)
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
    assert torch.cuda.is_available(), "the H100 stage-3 trainer needs a CUDA device (no CPU fallback)"
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

    # ---- models (:117-151) ----
    model = DVT.PretrainedViTWrapper(model_identifier=args.model, stride=args.stride_size)
    pos_h = (args.input_size[0] - model.patch_size) // args.stride_size + 1
    pos_w = (args.input_size[1] - model.patch_size) // args.stride_size + 1
    args.feat_dim = model.n_output_dims
    args.noise_map_height, args.noise_map_width = pos_h, pos_w
    normalizer = model.transformation.transforms[-1]
    assert isinstance(normalizer, transforms.Normalize), "last transform must be norm"

    pretrained_vit = DVT.PretrainedViTWrapper(model_identifier=args.model, stride=args.stride_size)
    teacher = DVT.Denoiser(noise_map_height=pos_h, noise_map_width=pos_w, feat_dim=args.feat_dim, vit=pretrained_vit,
                           num_blocks=args.num_blocks).to(device)
    msg = teacher.load_state_dict(torch.load(args.denoiser_ckpt, map_location="cpu")["denoiser"], strict=False)
    missing = {k for k in msg.missing_keys if "vit" not in k}
    print(f"Loaded denoiser from {args.denoiser_ckpt}; missing keys: {missing}, unexpected keys: {msg.unexpected_keys}")
    teacher.eval()
    for p in teacher.parameters():
        p.requires_grad_(False)

    model = model.to(device)
    model.set_trainable(True)
    if args.grad_checkpointing:
        print("Enable gradient checkpointing")
        model.model.set_grad_checkpointing(True)
    start_step = 0
    ck = None
    if args.resume:
        ck = torch.load(args.resume, map_location=device)
        model.load_state_dict(ck["model"], strict=True)
        start_step = int(ck["step"]) + 1
    if world > 1:  # every rank starts from rank 0's weights (what DistributedDataParallel does at construction)
        import torch.distributed as dist
        for p in model.parameters():
            dist.broadcast(p.data, 0)
    if rank == 0:
        print(f"Model = {model}")

    # ---- data (:152-186) ----
    train_dataset = ImageFolder(root=args.data_root, transform=transforms.Compose([
        transforms.Resize(args.input_size, interpolation=Image.BICUBIC, antialias=True),
        transforms.RandomHorizontalFlip(),
        transforms.ToTensor(),
        normalizer,
    ]))
    print(f"Dataset size: {len(train_dataset)}")
    sampler = (dataset.DistributedInfiniteSampler(train_dataset, num_replicas=world, rank=rank) if world > 1
               else dataset.InfiniteSampler(train_dataset))
    steps_per_epoch = len(train_dataset) // (args.batch_size * world)
    print(f"steps_per_epoch: {steps_per_epoch}")
    if args.num_iterations is None:
        args.num_iterations = steps_per_epoch * args.num_epochs
    data_loader = torch.utils.data.DataLoader(train_dataset, batch_size=args.batch_size, sampler=sampler,
                                              num_workers=args.num_workers, pin_memory=True, drop_last=False)

    # ---- optimiser and schedule (:187-205) ----
    args.lr = args.blr * math.sqrt(args.batch_size * world / 256)
    print(f"sqrt scaling learning rate; blr: {args.blr}, actual lr: {args.lr}")
    optimizer = FusedAdamW(model.parameters(), betas=(0.9, 0.999), weight_decay=args.weight_decay)
    sched = dict(base_value=args.lr, final_value=args.min_lr, total_iters=args.num_iterations,
                 warmup_iters=int(args.num_iterations * 0.15), start_warmup_value=0)
    if ck is not None:
        optimizer.load_state_dict(ck["optimizer"])
        print(f"Resumed from {args.resume} at step {start_step}")

    # ---- loop (:209-285) ----
    end = start = time.time()
    window = []
    it = iter(data_loader)
    for step in range(start_step, args.num_iterations):
        samples = next(it)[0].to(device, non_blocking=True)
        data_time = time.time() - end
        lr = misc.cosine_schedule(step, **sched)
        misc.apply_optim_scheduler(optimizer, lr)
        with torch.no_grad():
            target = teacher(samples, return_dict=True)["denoised_feats"]
        pred = model.get_intermediate_layers(samples)[0].permute(0, 2, 3, 1)
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
            iter_time = time.time() - end
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
