"""The NYU depth probe (reference evaluate_dense_tasks.py --task depth with vitb_nyu_linear_config.py: build_depther,
DepthEncoderDecoder, BNHead classify=True, SigLoss + GradientLoss, NYUDataset), trained and evaluated on the sm_90a
kernels of depth_ops, with what mmcv 1.x's IterBasedRunner runs for that config restated: AdamW with paramwise
custom_keys, gradient clipping, CosineAnnealing LR with linear warmup, OneCycle momentum, CheckpointHook with
max_keep_ckpts and EvalHook with save_best."""
from __future__ import annotations

import math
import os
import time
import warnings
from functools import partial
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
import torch.distributed as dist
import torch.nn as nn

from . import depth_ops
from .config import ConfigError
from .data import StreamSampler, worker_init_fn
from .depth_data import NYUDataset
from .model import ProbeBackbone, head_state_dict, in_channels_of, load_head_state_dict
from .trainer import JsonLog, _rank_world

METRICS = ("a1", "a2", "a3", "abs_rel", "rmse", "log_10", "rmse_log", "silog", "sq_rel")


# ---------------------------------------------------------------------------------------------------------------------
# schedules (mmcv 1.x hooks, by iteration, set before the step at 0-based iteration `it`)
# ---------------------------------------------------------------------------------------------------------------------
def annealing_cos(start: float, end: float, factor: float) -> float:
    return end + 0.5 * (start - end) * (math.cos(math.pi * factor) + 1)


def cosine_lr(it: int, base_lr: float, max_iters: int, min_lr_ratio: float = 0.0, warmup: Optional[str] = None,
              warmup_iters: int = 0, warmup_ratio: float = 0.1) -> float:
    """CosineAnnealingLrUpdaterHook(min_lr_ratio): regular = annealing_cos(base, base * min_lr_ratio, it / max_iters);
    during linear warmup (it < warmup_iters) regular * (1 - (1 - it / warmup_iters) (1 - warmup_ratio))."""
    regular = annealing_cos(base_lr, base_lr * min_lr_ratio, it / max_iters)
    if warmup is None or it >= warmup_iters:
        return regular
    return regular * (1 - (1 - it / warmup_iters) * (1 - warmup_ratio))


def one_cycle_momentum(it: int, max_iters: int, base_momentum: float = 0.85, max_momentum: float = 0.95,
                       pct_start: float = 0.3) -> float:
    """OneCycleMomentumUpdaterHook (two phases, cos): max -> base up to iteration pct_start * max_iters - 1, then back to
    max at max_iters - 1.  For AdamW it sets beta1."""
    phases = [(float(pct_start * max_iters) - 1, max_momentum, base_momentum), (max_iters - 1, base_momentum, max_momentum)]
    start = 0.0
    for i, (end, a, b) in enumerate(phases):
        if it <= end or i == len(phases) - 1:
            return annealing_cos(a, b, (it - start) / (end - start))
        start = end
    raise AssertionError


def param_groups(named_params, base_lr: float, weight_decay: float, custom_keys: Optional[dict]) -> List[dict]:
    """mmcv DefaultOptimizerConstructor with paramwise_cfg.custom_keys: one group per parameter; the longest key (ties:
    alphabetical) that is a substring of the parameter's name sets lr_mult / decay_mult."""
    keys = sorted(sorted(custom_keys or {}), key=len, reverse=True)
    groups = []
    for name, p in named_params:
        g = {"params": [p], "lr": base_lr, "weight_decay": weight_decay, "name": name}
        for key in keys:
            if key in name:
                g["lr"] = base_lr * custom_keys[key].get("lr_mult", 1.0)
                g["weight_decay"] = weight_decay * custom_keys[key].get("decay_mult", 1.0)
                break
        g["initial_lr"] = g["lr"]
        groups.append(g)
    return groups


# ---------------------------------------------------------------------------------------------------------------------
# head
# ---------------------------------------------------------------------------------------------------------------------
class DepthHead(nn.Module):
    """BNHead(classify=True, UD bins, linear norm) of the depth configs.  Despite the name it has no BatchNorm (the
    reference's is commented out): conv_depth is a 1x1 conv `channels` -> n_bins with PyTorch's default init, on
    cat(features, cls expanded) upsampled x `upsample`.  Here the conv runs at the feature grid and the kernel does the
    upsample and the bin expectation.  forward(feat NHWC [B, h, w, nC], cls [B, nC]) -> depth [B, h up, w up]."""

    def __init__(self, channels: int, n_bins: int, min_depth: float, max_depth: float, upsample: int, n_maps: int = 1):
        super().__init__()
        self.conv_depth = nn.Conv2d(channels, n_bins, kernel_size=1)
        self.min_depth, self.max_depth, self.upsample, self.n_maps = float(min_depth), float(max_depth), int(upsample), n_maps
        self.register_buffer("bins", torch.linspace(min_depth, max_depth, n_bins), persistent=False)

    def forward(self, feat: torch.Tensor, cls: torch.Tensor) -> torch.Tensor:
        logits = depth_ops.head_logits(feat, cls, self.conv_depth.weight, self.conv_depth.bias, self.n_maps)
        return depth_ops.bin_expectation(logits, self.bins, self.upsample)


def build_head(cfg: dict, backbone: ProbeBackbone, device) -> DepthHead:
    hc = cfg["model"]["decode_head"]
    chans = sum(in_channels_of(hc))
    if chans != backbone.channels or int(hc["channels"]) != 2 * backbone.channels:
        raise ValueError(f"decode_head in_channels {hc.get('in_channels')} / channels {hc.get('channels')} do not match the "
                         f"backbone's {backbone.channels} feature channels (+ as many cls channels); set them with "
                         f"--cfg-options model.decode_head.in_channels=[{backbone.channels}] "
                         f"model.decode_head.channels={2 * backbone.channels}")
    return DepthHead(int(hc["channels"]), int(hc.get("n_bins", 256)), hc.get("min_depth", 1e-3), hc["max_depth"],
                     int(hc.get("upsample", 1)), len(backbone.in_index)).to(device)


# ---------------------------------------------------------------------------------------------------------------------
# metrics
# ---------------------------------------------------------------------------------------------------------------------
def metrics_from_sums(s: Sequence[float]) -> np.ndarray:
    """The nine values of the reference's calculate() (a1, a2, a3, abs_rel, rmse, log_10, rmse_log, silog, sq_rel) from
    one image's dvt_depth_eval_sums: all NaN for an empty mask; silog NaN (a negative variance) becomes 0."""
    n, c1, c2, c3, ar, sr, d2, e, e2, l10 = (float(v) for v in s)
    if n == 0:
        return np.full(9, np.nan)
    with np.errstate(invalid="ignore"):
        silog = float(np.sqrt(e2 / n - (e / n) ** 2) * 100)
    if np.isnan(silog):
        silog = 0.0
    return np.array([c1 / n, c2 / n, c3 / n, ar / n, math.sqrt(d2 / n), l10 / n, math.sqrt(e2 / n), silog, sr / n])


def gather_rows(indices: Sequence[int], rows: np.ndarray, n_total: int) -> np.ndarray:
    """This rank's per-image metric rows [len(indices), 9] -> every rank's, [n_total, 9] in dataset order."""
    rows = np.asarray(rows, dtype=np.float64).reshape(-1, 9)
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        parts = [None] * dist.get_world_size()
        dist.all_gather_object(parts, (list(indices), rows))
    else:
        parts = [(list(indices), rows)]
    out = np.full((n_total, 9), np.nan)
    seen = np.zeros(n_total, dtype=bool)
    for idx, r in parts:
        out[idx] = r
        seen[idx] = True
    if not seen.all():
        raise RuntimeError(f"depth evaluation: images {np.nonzero(~seen)[0][:8].tolist()} were evaluated by no rank")
    return out


def summarize(rows: np.ndarray) -> Dict[str, float]:
    """nanmean over images of each metric (pre_eval_to_metrics)."""
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        means = np.nanmean(rows, axis=0)
    return {k: float(v) for k, v in zip(METRICS, means)}


@torch.no_grad()
def evaluate(backbone: ProbeBackbone, head: DepthHead, dataset: NYUDataset, device, workers: int = 0) -> Dict[str, float]:
    """Whole inference of this rank's share of the validation set (images rank, rank + world, ...): each image's
    augmentations go through the backbone and head as one batch, then dvt_depth_eval_sums; the per-image metric rows of
    all ranks are gathered and averaged in dataset order."""
    rank, world = _rank_world()
    mine = list(range(rank, len(dataset), world))
    loader = torch.utils.data.DataLoader(
        torch.utils.data.Subset(dataset, mine), batch_size=None, num_workers=workers, pin_memory=True,
        worker_init_fn=partial(worker_init_fn, num_workers=workers, rank=rank, seed=0) if workers > 0 else None)
    sums = torch.zeros(len(mine), 10, dtype=torch.float64, device=device)
    ws = torch.empty(depth_ops.EVAL_WORKSPACE, dtype=torch.float64, device=device)
    for j, (augs, gt) in enumerate(loader):
        imgs = torch.stack([a for a, _ in augs]).to(device, non_blocking=True)
        gt = gt.to(device, non_blocking=True)
        maps = head(*backbone(imgs))
        depth_ops.eval_sums(maps, [bool(f) for _, f in augs], gt, dataset.min_depth, dataset.max_depth,
                            dataset.eval_crop(*gt.shape), sums[j], ws)
    rows = np.stack([metrics_from_sums(s) for s in sums.cpu().numpy()]) if mine else np.zeros((0, 9))
    return summarize(gather_rows(mine, rows, len(dataset)))


# ---------------------------------------------------------------------------------------------------------------------
# training
# ---------------------------------------------------------------------------------------------------------------------
def depth_losses(pred4: torch.Tensor, gt: torch.Tensor, sig: depth_ops.SigLossState, sig_weight: float = 1.0,
                 grad_weight: float = 0.5) -> dict:
    """decode.loss_depth, decode.loss_grad and their sum, from the head's depth at the upsampled grid and gt [B, H, W]."""
    pred = depth_ops.resize(pred4, gt.shape[-2:])[:, None]
    gt = gt[:, None]
    ld = sig_weight * sig(pred, gt)
    lg = grad_weight * depth_ops.gradient_loss(pred, gt)
    return {"decode.loss_depth": ld, "decode.loss_grad": lg, "loss": ld + lg}


def _loss_cfg(cfg: dict, kind: str) -> dict:
    return next(l for l in cfg["model"]["decode_head"]["loss_decode"] if l["type"] == kind)


def _save(path: str, head, opt, n: int, meta: dict) -> None:
    torch.save({"state_dict": head_state_dict(head), "optimizer": opt.state_dict(), "iter": n, "meta": meta}, path)


def train(cfg: dict, backbone_model, work_dir: str, seed: int, device, validate: bool = True,
          resume_from: Optional[str] = None, timestamp: Optional[str] = None, exp_name: str = "") -> dict:
    rank, world = _rank_world()
    bc, hc = cfg["model"]["backbone"], cfg["model"]["decode_head"]
    backbone = ProbeBackbone(backbone_model, bc["out_indices"], hc["in_index"], return_cls=True,
                             norm=bool(bc.get("final_norm", False)))
    if backbone.is_denoiser and list(hc["in_index"]) != [0]:
        raise ConfigError(f"decode_head in_index {hc['in_index']}: the Denoiser backbone gives one map (in_index [0])")
    torch.manual_seed(seed)
    head = build_head(cfg, backbone, device)
    oc = cfg["optimizer"]
    groups = param_groups([("decode_head." + n, p) for n, p in head.named_parameters()], oc["lr"],
                          oc.get("weight_decay", 1e-2), (oc.get("paramwise_cfg") or {}).get("custom_keys"))
    opt = torch.optim.AdamW(groups, lr=oc["lr"], betas=tuple(oc.get("betas", (0.9, 0.999))), eps=oc.get("eps", 1e-8),
                            weight_decay=oc.get("weight_decay", 1e-2))
    start, best_score, best_ckpt = 0, math.inf, None
    if resume_from is not None:
        ck = torch.load(resume_from, map_location=device)
        load_head_state_dict(head, ck["state_dict"])
        opt.load_state_dict(ck["optimizer"])
        start = int(ck["iter"])
        best_score = ck.get("meta", {}).get("best_score", math.inf)
        best_ckpt = ck.get("meta", {}).get("best_ckpt")
    model = head
    if world > 1:
        model = torch.nn.parallel.DistributedDataParallel(head, device_ids=[device.index])

    data = cfg["data"]
    batch, workers = int(data["samples_per_gpu"]), int(data.get("workers_per_gpu", 0))
    max_iters = int(cfg["runner"]["max_iters"])
    lr_cfg = cfg["lr_config"]
    sched = dict(max_iters=max_iters, min_lr_ratio=lr_cfg.get("min_lr_ratio", 0.0), warmup=lr_cfg.get("warmup"),
                 warmup_iters=lr_cfg.get("warmup_iters", 0), warmup_ratio=lr_cfg.get("warmup_ratio", 0.1))
    mom_cfg = cfg.get("momentum_config")
    clip = (cfg.get("optimizer_config") or {}).get("grad_clip")
    ck_cfg = cfg.get("checkpoint_config", {})
    ckpt_interval, max_keep = int(ck_cfg.get("interval", max_iters)), int(ck_cfg.get("max_keep_ckpts", -1))
    ev_cfg = cfg.get("evaluation", {})
    eval_interval, key = int(ev_cfg.get("interval", max_iters)), ev_cfg.get("save_best")
    better = (lambda a, b: a > b) if ev_cfg.get("rule", "less") == "greater" else (lambda a, b: a < b)
    if best_score == math.inf and ev_cfg.get("rule") == "greater":
        best_score = -math.inf
    log_interval = int(cfg.get("log_config", {}).get("interval", 50))
    sl = _loss_cfg(cfg, "SigLoss")
    sig = depth_ops.SigLossState(bool(sl.get("warm_up", False)), int(sl.get("warm_iter", 100)))
    sig_weight = float(sl.get("loss_weight", 1.0))
    grad_weight = float(_loss_cfg(cfg, "GradientLoss").get("loss_weight", 1.0))

    train_set = NYUDataset(data["train"], train=True, seed=seed)
    val_set = NYUDataset(data["val"], train=False) if validate else None
    loader = torch.utils.data.DataLoader(
        train_set, batch_size=batch, sampler=StreamSampler(start, max_iters, batch, rank, world), num_workers=workers,
        pin_memory=True, drop_last=True,
        worker_init_fn=partial(worker_init_fn, num_workers=workers, rank=rank, seed=seed) if workers > 0 else None)
    log = JsonLog(os.path.join(work_dir, f"{timestamp or time.strftime('%Y%m%d_%H%M%S')}.log.json") if rank == 0 else None)
    log.write({"exp_name": exp_name, "seed": seed, "world_size": world, "start_iter": start, "max_iters": max_iters})
    last_eval, window = None, []
    t0 = time.time()
    model.train()
    for it, (img, gt) in zip(range(start, max_iters), loader):
        for g in opt.param_groups:
            g["lr"] = cosine_lr(it, g["initial_lr"], **sched)
            if mom_cfg is not None:
                g["betas"] = (one_cycle_momentum(it, max_iters), g["betas"][1])
        img, gt = img.to(device, non_blocking=True), gt.to(device, non_blocking=True)
        feat, cls = backbone(img)
        losses = depth_losses(model(feat, cls), gt, sig, sig_weight, grad_weight)
        opt.zero_grad(set_to_none=True)
        losses["loss"].backward()
        if clip is not None:
            torch.nn.utils.clip_grad_norm_([p for p in head.parameters() if p.grad is not None], clip["max_norm"],
                                           clip.get("norm_type", 2))
        opt.step()
        window.append(torch.stack([losses[k].detach() for k in ("decode.loss_depth", "decode.loss_grad", "loss")]))
        n = it + 1
        if n % log_interval == 0 or n == max_iters:
            vals = torch.stack(window).mean(0).tolist()     # the only host synchronisation of the step loop
            window = []
            if not math.isfinite(vals[2]):
                raise FloatingPointError(f"loss is {vals[2]} at iteration {n}")
            lr = opt.param_groups[0]["lr"]
            if rank == 0:
                print(f"Iter [{n}/{max_iters}] lr: {lr:.4e}, decode.loss_depth: {vals[0]:.4f}, decode.loss_grad: "
                      f"{vals[1]:.4f}, loss: {vals[2]:.4f}, time: {time.time() - t0:.1f}s", flush=True)
            log.write({"mode": "train", "iter": n, "lr": lr, "momentum": opt.param_groups[0]["betas"][0],
                       "decode.loss_depth": vals[0], "decode.loss_grad": vals[1], "loss": vals[2]})
        meta = {"seed": seed, "exp_name": exp_name, "best_score": best_score, "best_ckpt": best_ckpt}
        if rank == 0 and (n % ckpt_interval == 0 or n == max_iters):
            path = os.path.join(work_dir, f"iter_{n}.pth")
            _save(path, head, opt, n, meta)
            latest = os.path.join(work_dir, "latest.pth")
            if os.path.lexists(latest):
                os.remove(latest)
            os.symlink(os.path.basename(path), latest)
            if max_keep > 0:     # CheckpointHook: drop iter_<n - k interval> for k >= max_keep, newest first
                for step in range(n - max_keep * ckpt_interval, 0, -ckpt_interval):
                    old = os.path.join(work_dir, f"iter_{step}.pth")
                    if not os.path.exists(old):
                        break
                    os.remove(old)
        if validate and n % eval_interval == 0:
            res = evaluate(backbone, head, val_set, device, workers)
            last_eval = dict(res, iter=n)
            if rank == 0:
                print(f"Iter(val) [{n}] " + ", ".join(f"{k}: {res[k]:.4f}" for k in METRICS), flush=True)
            log.write(dict(mode="val", **last_eval))
            if key is not None and better(res[key], best_score):
                best_score = res[key]
                if rank == 0:
                    if best_ckpt is not None and os.path.exists(os.path.join(work_dir, best_ckpt)):
                        os.remove(os.path.join(work_dir, best_ckpt))
                    best_ckpt = f"best_{key}_iter_{n}.pth"
                    _save(os.path.join(work_dir, best_ckpt), head, opt, n,
                          dict(meta, best_score=best_score, best_ckpt=best_ckpt))
    torch.cuda.synchronize(device)
    return {"head": head, "last_eval": last_eval, "sig_loss_calls": sig.counter}
