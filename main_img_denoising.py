"""DVT stage 1 (per-image denoising) on H100 -- drop-in for the reference's main_img_denoising.py.

Same command line (reference main_img_denoising.py:152-217), same outputs
(`{save_root}/raw_features/{model}/<rel>.npy` (h, w, C) float32 and `{save_root}/denoised_features/{model}/<rel>.npy`
(1, h, w, C) float32, :131-146), same skip/resume rule (:303-307).  The two hot paths run in libdvt_b200.so:
feature-bank extraction (769 ViT forwards) and the neural-field fit (`denoise_an_image`).

How the loop differs from the reference's (one image after the other, everything synchronous):
  * images are software-pipelined (`Stage1Pipeline.run_images`): the host only enqueues; the views of image i+1 are cut
    (on the GPU) and its bank is extracted while image i is being fitted; results are collected one image late;
  * the `.npy` files are written by a background thread from pinned staging buffers (`dvt.store.FeatureStoreWriter`);
  * under `torchrun` (WORLD_SIZE > 1) the image list is sharded rank-strided -- the reference starts 8 unrelated
    processes over index ranges, sample_scripts/stage1.sh:8-19 -- and the denoised maps are collated on every rank with
    ONE NCCL all-gather (`dvt.dist.collate_maps`), ready for stage 2 without the disk hand-off (`--collate_out` keeps
    the gathered stack on rank 0).

Deliberate differences, documented in DESIGN.md: the PCA visualisation of every `vis_freq`-th image (reference
:101-117) is not produced (matplotlib / torch_kmeans are outside the hot path; the RNG draw it makes is still made, so
the sampling streams of later images stay those of the reference); `--dtype` selects the element type of the generated
views (the ViT kernels always compute bf16 x bf16 -> fp32, the fit in 3xTF32).
"""
import argparse
import datetime
import glob
import json
import os
import sys
import time

import numpy as np
import torch
from torchvision import transforms

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "denoising-vit_b200"))

import dvt.models as DVT  # noqa: E402
import dvt.utils.misc as misc  # noqa: E402
from dvt import dist as dvt_dist  # noqa: E402
from dvt.dataset import GpuViewGenerator, load_image  # noqa: E402
from dvt.stage1 import Stage1Config, Stage1Pipeline  # noqa: E402
from dvt.store import FeatureStoreWriter  # noqa: E402


def print_losses(args, losses: np.ndarray):
    """The lines the reference prints during the loop (main_img_denoising.py:91-100), from the per-step loss table."""
    for step in sorted(set(list(range(0, args.num_iters, 1000)) + [args.num_iters - 1])):
        lr = misc.learning_rate_at(step, args.lr, args.min_lr, args.warmup_iters, args.num_iters)
        l = losses[step]
        print(f"Step {step}/{args.num_iters - 1}: Loss = {l[0]:.4f}, Patch Loss = {l[1]:.4f}, CosSim Loss = {l[2]:.4f}, "
              f"Residual Loss = {l[3]:.4f}, Residual Sparsity Loss = {l[4]:.4f}, LR = {lr:.4f}")


def draw_sampling_stream(args, n_rows: int, image_index: int) -> np.ndarray:
    """The reference draws np.random.randint(0, n_rows, pixel_bsz) once per step from the global legacy RNG (:73) and,
    for every `vis_freq`-th image, np.random.randint(0, num_views + 1, num_vis_samples) after the loop (:102).  Drawing
    all steps at once, as int32, consumes the identical MT19937 stream (checked in tests/test_store_cpu.py)."""
    idx = np.random.randint(0, n_rows, (args.num_iters, args.pixel_bsz), dtype=np.int32)
    if image_index % args.vis_freq == 0:
        np.random.randint(0, args.num_views + 1, args.num_vis_samples)
    return idx


def get_args(argv=None):
    p = argparse.ArgumentParser(description="DVT Stage-1: Single Image Denoising")
    p.add_argument("--model", type=str, default="vit_base_patch14_dinov2.lvd142m", choices=DVT.MODEL_LIST)
    p.add_argument("--input_size", type=int, default=518, nargs="+")
    p.add_argument("--stride_size", type=int, default=14)
    p.add_argument("--layer_depth_ratio", type=float, default=1.0)
    p.add_argument("--img_path", type=str, default="demo/assets/demo/cat.jpg")
    p.add_argument("--dtype", type=str, default="float32")
    p.add_argument("--data_root", type=str, default=None)
    p.add_argument("--save_root", type=str, default=None)
    p.add_argument("--start_idx", type=int, default=0)
    p.add_argument("--num_imgs", type=int, default=100)
    p.add_argument("--num_views", type=int, default=768)
    p.add_argument("--num_iters", type=int, default=25000)
    p.add_argument("--warmup_iters", type=int, default=2500)
    p.add_argument("--n_levels", type=int, default=16)
    p.add_argument("--freeze_shared_artifacts_after", type=float, default=0.5)
    p.add_argument("--lr", type=float, default=0.01)
    p.add_argument("--min_lr", type=float, default=0.001)
    p.add_argument("--weight_decay", type=float, default=1e-5)
    p.add_argument("--extract_bsz", type=int, default=32)
    p.add_argument("--pixel_bsz", type=int, default=2048)
    p.add_argument("--output_dir", type=str, default="./work_dirs/demo")
    p.add_argument("--num_vis_samples", type=int, default=5)
    p.add_argument("--vis_freq", type=int, default=100)
    p.add_argument("--seed", type=int, default=0)
    # H100 extensions (not reference flags)
    p.add_argument("--collate_out", type=str, default=None,
                   help="rank 0 saves the all-gathered stacks of raw and denoised maps [N, h, w, C] (+ the image list) here "
                        "(.pt); main_denoiser.py --collated trains from it")
    p.add_argument("--sequential", action="store_true", help="one image after the other (no pipelining over images)")
    args = p.parse_args(argv)
    assert os.path.exists(args.img_path), f"Image not found: {args.img_path}"
    if isinstance(args.input_size, int):
        args.input_size = (args.input_size, args.input_size)
    elif len(args.input_size) == 1:
        args.input_size = (args.input_size[0], args.input_size[0])
    args.input_size = tuple(args.input_size)
    assert args.input_size[0] % args.stride_size == 0, "height must be divisible by stride_size"
    assert args.input_size[1] % args.stride_size == 0, "width must be divisible by stride_size"
    return args


def main(args):
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    os.makedirs(args.output_dir, exist_ok=True)
    misc.fix_random_seeds(args.seed)
    if rank == 0:
        print(f"Arguments:\n{json.dumps(vars(args), indent=4)}")
    assert torch.cuda.is_available(), "the H100 stage-1 driver needs a CUDA device (no CPU fallback)"
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=device)
    if os.path.isfile(args.img_path):
        if args.img_path.endswith("txt"):
            with open(args.img_path) as f:
                filenames = f.read().splitlines()
        else:
            filenames = [args.img_path]
    else:
        filenames = sorted(glob.glob(os.path.join(args.img_path, "**/*"), recursive=True))
    filenames = filenames[args.start_idx:args.start_idx + args.num_imgs]

    vit = DVT.PretrainedViTWrapper(model_identifier=args.model, stride=args.stride_size).to(device).eval()
    layer_index = int(args.layer_depth_ratio * vit.last_layer_index)
    args.layer_index, args.feat_dim = layer_index, vit.n_output_dims
    normalizer = vit.transformation.transforms[-1]
    assert isinstance(normalizer, transforms.Normalize), "last transform must be norm"
    view_dtype = torch.float32 if args.dtype == "float32" else torch.bfloat16
    cfg = Stage1Config(num_iters=args.num_iters, warmup_iters=args.warmup_iters, n_levels=args.n_levels,
                       freeze_shared_artifacts_after=args.freeze_shared_artifacts_after, lr=args.lr, min_lr=args.min_lr,
                       weight_decay=args.weight_decay, extract_bsz=args.extract_bsz, pixel_bsz=args.pixel_bsz,
                       log_losses=True)
    pipe = Stage1Pipeline(vit, layer_index, args.input_size, cfg, seed=args.seed)
    args.noise_map_height, args.noise_map_width = pipe.h, pipe.w

    # ---- work list: (position in the list, path); finished images are skipped (reference :303-307) ----
    todo = []
    for idx, filename in enumerate(filenames):
        filename = filename.strip().split(" ")[0]
        if args.data_root is not None:
            filename = os.path.join(args.data_root, filename)
            if misc.check_if_file_exists(args, filename):
                if rank == 0:
                    print(f"Skipping {filename}")
                continue
        todo.append((idx, filename))
    mine = [todo[k] for k in dvt_dist.shard_indices(len(todo), rank, world)]

    num_samples = args.num_views + 1  # + the un-augmented image
    n_rows = num_samples * pipe.h * pipe.w
    view_gen = GpuViewGenerator(args.input_size, num_views=args.num_views, scale=(0.1, 0.5), patch_size=vit.patch_size,
                                stride=args.stride_size, dtype=view_dtype,
                                flip_rng=np.random.RandomState(args.seed + 7919 * (rank + 1)))
    views_dev = torch.empty((num_samples, 3) + args.input_size, dtype=view_dtype, device=device)
    coords_of = {}
    img_pinned = [torch.empty((3,) + args.input_size, dtype=torch.float32).pin_memory() for _ in range(2)]
    img_copied = [torch.cuda.Event(), torch.cuda.Event()]
    writer = FeatureStoreWriter() if args.data_root is not None else None
    keep_maps = world > 1 or args.collate_out is not None
    maps = []
    start = time.time()
    state = {"done": 0, "last": start}

    def views_fn(i):
        # host: decode + resize + normalise one image (overlaps the GPU work of the previous images); device: all views
        # of the image in one launch.  `views_dev` is reused: the launch is ordered behind the forwards that read it.
        # The image goes through a pinned staging buffer: a pageable copy would block the host until the stream has drained.
        img_copied[i % 2].synchronize()
        img_pinned[i % 2].copy_(load_image(mine[i][1], args.input_size, normalizer.mean, normalizer.std))
        image = img_pinned[i % 2].to(device, non_blocking=True)
        img_copied[i % 2].record()
        views, coords = view_gen(image, views_out=views_dev)
        coords_of[i] = coords
        return views

    def finalize(i, out):
        idx, filename = mine[i]
        out["losses_ready"].synchronize()            # the fit of this image has finished (the next one is already queued)
        print_losses(args, out["losses"].numpy())
        if writer is not None:
            raw_path, den_path = misc.feature_paths(args, filename)
            writer.submit(raw_path, den_path, out["raw"], out["denoised_feats"])
            print(f"Saving denoised features to {den_path} and raw features to {raw_path}")
        if keep_maps:
            maps.append(torch.stack([out["raw"], out["denoised_feats"][0]]))     # [2, h, w, C]: the stage-2 training pair
        coords_of.pop(i, None)
        now = time.time()
        state["done"] += 1
        eta = (now - start) / state["done"] * (len(mine) - state["done"])
        print(f"[{idx + 1}/{len(filenames)}] {filename}: {now - state['last']:.2f}s, "
              f"ETA: {datetime.timedelta(seconds=int(eta))}, Elapsed: {datetime.timedelta(seconds=int(now - start))}")
        print("-" * 80)
        state["last"] = now
        return filename

    pipe.run_images(len(mine), views_fn, lambda i: coords_of[i], lambda i: draw_sampling_stream(args, n_rows, mine[i][0]),
                    finalize, overlap=not args.sequential)
    if writer is not None:
        writer.close()
    if keep_maps:
        local_maps = (torch.stack(maps) if maps else
                      torch.empty((0, 2, pipe.h, pipe.w, pipe.C), device=device, dtype=torch.float32))
        gathered = dvt_dist.collate_maps(local_maps, len(todo))       # the single exchange of the path (NCCL all-gather)
        if rank == 0:
            print(f"Collated raw + denoised maps of {gathered.shape[0]} images on every rank: {tuple(gathered.shape)}")
            if args.collate_out is not None:
                torch.save({"raw_feats": gathered[:, 0].cpu(), "denoised_feats": gathered[:, 1].cpu(),
                            "files": [f for _, f in todo], "model": args.model}, args.collate_out)
    torch.cuda.synchronize()
    print(f"Total time: {datetime.timedelta(seconds=int(time.time() - start))}")
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main(get_args())
