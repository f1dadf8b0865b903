"""Iteration-based trainer of the segmentation probe (what mmseg's train_segmentor runs for the linear configs: mmcv
IterBasedRunner, PolyLrUpdaterHook with linear warmup, AdamW on the head, CheckpointHook, EvalHook)."""
from __future__ import annotations

import json
import math
import os
import time
from functools import partial
from typing import Optional

import numpy as np
import torch
import torch.distributed as dist

from . import seg_ops
from .data import SegDataset, StreamSampler, worker_init_fn
from .metrics import metrics_from_hist
from .model import LinearSegHead, ProbeBackbone, head_state_dict, in_channels_of, load_head_state_dict


def poly_lr(it: int, base_lr: float, max_iters: int, power: float = 1.0, min_lr: float = 0.0, warmup: Optional[str] = None,
            warmup_iters: int = 0, warmup_ratio: float = 0.1) -> float:
    """mmcv 1.x PolyLrUpdaterHook (by_epoch=False) at 0-based iteration `it`, set before the step:
    regular = (base - min) (1 - it / max)^power + min; during linear warmup (it < warmup_iters)
    regular * (1 - (1 - it / warmup_iters) (1 - warmup_ratio))."""
    regular = (base_lr - min_lr) * (1 - it / max_iters) ** power + min_lr
    if warmup is None or it >= warmup_iters:
        return regular
    return regular * (1 - (1 - it / warmup_iters) * (1 - warmup_ratio))


def _rank_world():
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


class JsonLog:
    def __init__(self, path: Optional[str]):
        self.path = path

    def write(self, rec: dict):
        if self.path is not None:
            with open(self.path, "a") as fh:
                fh.write(json.dumps(rec) + "\n")


@torch.no_grad()
def evaluate(backbone: ProbeBackbone, head: LinearSegHead, dataset: SegDataset, test_cfg: dict, num_classes: int,
             device, workers: int = 0) -> dict:
    """Slide inference over this rank's share of the validation set (images rank, rank + world, ...), decoded and resized
    by `workers` DataLoader workers (results in index order), histograms summed over ranks (exact int64 all-reduce),
    metrics from the totals.  A test pipeline with several augmentations (multi-scale / flip) runs mmseg's aug_test."""
    rank, world = _rank_world()
    was_training = head.training
    head.eval()
    hist = torch.zeros(4, num_classes, dtype=torch.int64, device=device)
    fn = lambda crops: head(backbone(crops))  # noqa: E731
    share = torch.utils.data.Subset(dataset, list(range(rank, len(dataset), world)))
    loader = torch.utils.data.DataLoader(
        share, batch_size=None, num_workers=workers, pin_memory=True,
        worker_init_fn=partial(worker_init_fn, num_workers=workers, rank=rank, seed=0) if workers > 0 else None)
    for img, gt in loader:
        gt = gt.to(device, non_blocking=True)
        if len(dataset.augs) > 1:       # mmseg aug_test: img is [(image, flip)] per augmentation
            augs = [(a.to(device, non_blocking=True), bool(flip)) for a, flip in img]
            seg_ops.aug_slide_inference_hist(fn, augs, gt, num_classes, test_cfg["crop_size"], test_cfg["stride"], hist)
        else:
            seg_ops.slide_inference_hist(fn, img.to(device, non_blocking=True), gt, num_classes, test_cfg["crop_size"],
                                         test_cfg["stride"], hist)
    if world > 1:
        dist.all_reduce(hist)
    head.train(was_training)
    return metrics_from_hist(hist.cpu().numpy())


def train(cfg: dict, backbone_model, work_dir: str, seed: int, device, validate: bool = True,
          resume_from: Optional[str] = None, timestamp: Optional[str] = None, exp_name: str = "") -> dict:
    rank, world = _rank_world()
    head_cfg = cfg["model"]["decode_head"]
    num_classes = int(head_cfg["num_classes"])
    backbone = ProbeBackbone(backbone_model, cfg["model"]["backbone"]["out_indices"], head_cfg["in_index"])
    if sum(in_channels_of(head_cfg)) != backbone.channels or head_cfg.get("channels", backbone.channels) != backbone.channels:
        raise ValueError(f"decode_head in_channels {head_cfg.get('in_channels')} / channels {head_cfg.get('channels')} do not "
                         f"match the backbone's {backbone.channels} feature channels; set them with --cfg-options "
                         f"model.decode_head.in_channels=[{backbone.channels}] model.decode_head.channels={backbone.channels}")
    torch.manual_seed(seed)
    head = LinearSegHead(backbone.channels, num_classes).to(device)
    if world > 1:
        head = torch.nn.SyncBatchNorm.convert_sync_batchnorm(head)
    oc = cfg["optimizer"]
    opt = torch.optim.AdamW(head.parameters(), lr=oc["lr"], betas=tuple(oc.get("betas", (0.9, 0.999))),
                            eps=oc.get("eps", 1e-8), weight_decay=oc.get("weight_decay", 1e-2))
    start = 0
    if resume_from is not None:
        ck = torch.load(resume_from, map_location=device)
        load_head_state_dict(head, ck["state_dict"])
        opt.load_state_dict(ck["optimizer"])
        start = int(ck["iter"])
    model = head
    if world > 1:
        model = torch.nn.parallel.DistributedDataParallel(head, device_ids=[device.index])

    data = cfg["data"]
    batch = int(data["samples_per_gpu"])
    workers = int(data.get("workers_per_gpu", 0))
    max_iters = int(cfg["runner"]["max_iters"])
    lr_cfg = cfg["lr_config"]
    sched = dict(base_lr=oc["lr"], max_iters=max_iters, power=lr_cfg.get("power", 1.0), min_lr=lr_cfg.get("min_lr", 0.0),
                 warmup=lr_cfg.get("warmup"), warmup_iters=lr_cfg.get("warmup_iters", 0),
                 warmup_ratio=lr_cfg.get("warmup_ratio", 0.1))
    ckpt_interval = int(cfg.get("checkpoint_config", {}).get("interval", max_iters))
    eval_interval = int(cfg.get("evaluation", {}).get("interval", max_iters))
    log_interval = int(cfg.get("log_config", {}).get("interval", 50))
    test_cfg = cfg["model"].get("test_cfg", cfg.get("test_cfg"))

    train_set = SegDataset(data["train"], num_classes, train=True, seed=seed)
    val_set = SegDataset(data["val"], num_classes, train=False) if validate else None
    loader = torch.utils.data.DataLoader(
        train_set, batch_size=batch, sampler=StreamSampler(start, max_iters, batch, rank, world), num_workers=workers,
        pin_memory=True, drop_last=True,
        worker_init_fn=partial(worker_init_fn, num_workers=workers, rank=rank, seed=seed) if workers > 0 else None)
    log = JsonLog(os.path.join(work_dir, f"{timestamp or time.strftime('%Y%m%d_%H%M%S')}.log.json") if rank == 0 else None)
    log.write({"exp_name": exp_name, "seed": seed, "world_size": world, "start_iter": start, "max_iters": max_iters})
    last_eval = None
    window = []
    t0 = time.time()
    model.train()
    for it, (img, seg) in zip(range(start, max_iters), loader):
        lr = poly_lr(it, **sched)
        for g in opt.param_groups:
            g["lr"] = lr
        img = img.to(device, non_blocking=True)
        seg = seg.to(device, non_blocking=True)
        feats = backbone(img)
        loss = seg_ops.upsample_cross_entropy(model(feats), seg)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
        window.append(loss.detach())
        n = it + 1
        if n % log_interval == 0 or n == max_iters:
            val = torch.stack(window).mean().item()     # the only host synchronisation of the step loop
            window = []
            if not math.isfinite(val):
                raise FloatingPointError(f"loss is {val} at iteration {n}")
            if rank == 0:
                print(f"Iter [{n}/{max_iters}] lr: {lr:.4e}, loss: {val:.4f}, time: {time.time() - t0:.1f}s", flush=True)
            log.write({"mode": "train", "iter": n, "lr": lr, "loss": val})
        if rank == 0 and (n % ckpt_interval == 0 or n == max_iters):
            path = os.path.join(work_dir, f"iter_{n}.pth")
            torch.save({"state_dict": head_state_dict(head), "optimizer": opt.state_dict(), "iter": n,
                        "meta": {"seed": seed, "exp_name": exp_name}}, path)
            latest = os.path.join(work_dir, "latest.pth")
            if os.path.lexists(latest):
                os.remove(latest)
            os.symlink(os.path.basename(path), latest)
        if validate and n % eval_interval == 0:
            res = evaluate(backbone, head, val_set, test_cfg, num_classes, device, workers)
            last_eval = dict(res, iter=n)
            if rank == 0:
                print(f"Iter(val) [{n}] aAcc: {res['aAcc']:.4f}, mIoU: {res['mIoU']:.4f}, mAcc: {res['mAcc']:.4f}",
                      flush=True)
            log.write(dict(mode="val", **last_eval))
    torch.cuda.synchronize(device)
    return {"head": head, "last_eval": last_eval}
