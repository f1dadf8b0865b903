"""Command-line set-up shared by evaluate_dense_tasks.py and evaluate_depth.py (the reference's evaluate_dense_tasks.py
main): config loading with --cfg-options / --options, work dir and resume rules, the launcher (one process, or torchrun
with NCCL), mmseg's init_random_seed and the --deterministic switch."""
from __future__ import annotations

import os
import os.path as osp
import random
import time
import warnings
from typing import Callable, Optional, Tuple

import numpy as np
import torch

from .config import load_config, merge_options


def load_run_config(args, check: Callable[[dict], None]) -> Tuple[dict, Optional[str]]:
    """The config with --cfg-options then --options merged, checked by `check`, with work_dir set; and the checkpoint to
    resume from (--resume-from, else the config's resume_from, else latest.pth under --auto-resume)."""
    cfg = load_config(args.config)
    if args.cfg_options is not None:
        merge_options(cfg, args.cfg_options)
    if args.options is not None:
        warnings.warn("--options is deprecated in favor of --cfg-options")
        merge_options(cfg, args.options)
    check(cfg)
    if args.work_dir is not None:
        cfg["work_dir"] = args.work_dir
    elif cfg.get("work_dir") is None:
        cfg["work_dir"] = osp.join("./work_dirs", osp.splitext(osp.basename(args.config))[0])
    resume_from = args.resume_from if args.resume_from is not None else cfg.get("resume_from")
    if resume_from is None and args.auto_resume and osp.exists(osp.join(cfg["work_dir"], "latest.pth")):
        resume_from = osp.join(cfg["work_dir"], "latest.pth")
    return cfg, resume_from


def init_run(args, cfg: dict, what: str):
    """Device, process group, work dir, seed and determinism of a run -> (rank, world, device, seed, timestamp)."""
    assert torch.cuda.is_available(), f"the H100 {what} needs a CUDA device (no CPU fallback)"
    import torch.distributed as dist
    if args.launcher == "none":
        rank, world, local = 0, 1, 0
    elif args.launcher == "pytorch":
        if "RANK" not in os.environ or "WORLD_SIZE" not in os.environ:
            raise RuntimeError("--launcher pytorch runs under torchrun (RANK / WORLD_SIZE are not set); use --launcher none "
                               "for one process")
        rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    else:
        raise NotImplementedError(f"--launcher {args.launcher}: only none and pytorch (torchrun) are implemented")
    torch.cuda.set_device(local)
    device = torch.device("cuda", local)
    if args.launcher == "pytorch":
        dist.init_process_group(cfg.get("dist_params", {}).get("backend", "nccl"), device_id=device)
    os.makedirs(osp.abspath(cfg["work_dir"]), exist_ok=True)
    timestamp = time.strftime("%Y%m%d_%H%M%S", time.localtime())

    # init_random_seed: a random seed is drawn on rank 0 and shared; --diff_seed adds the rank
    seed = args.seed
    if seed is None:
        t = torch.tensor([np.random.randint(2 ** 31)], dtype=torch.int64, device=device)
        if world > 1:
            dist.broadcast(t, 0)
        seed = int(t.item())
    if args.diff_seed:
        seed += rank
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    torch.cuda.manual_seed_all(seed)
    if args.deterministic:
        os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
        torch.use_deterministic_algorithms(True)
        torch.backends.cudnn.benchmark = False
    elif cfg.get("cudnn_benchmark", False):
        torch.backends.cudnn.benchmark = True
    if rank == 0:
        print(f"Set random seed to {seed}, deterministic: {args.deterministic}; work dir {cfg['work_dir']}", flush=True)
    return rank, world, device, seed, timestamp


def finish_run(world: int) -> None:
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()
