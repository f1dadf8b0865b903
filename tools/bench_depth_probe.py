"""Depth probe: the sm_90a head / loss / evaluation path against a torch restatement of the reference (features
upsampled x4, 1x1 conv at full resolution, relu + 0.1, normalise, einsum, F.interpolate, boolean-indexed SigLoss and
GradientLoss), both arms alternating in one process on one GPU.

Training step: ViT-B/14 with random weights (frozen, the same forward for both arms), 416 x 544 crops, batch 2 and 8:
step ms (median and range of three rounds), the two arms' loss difference and peak memory.  Evaluation: images/s at
480 x 640 with flip TTA (two augmentations), metrics included.  Prints the card name and power limit with the results.

    python tools/bench_depth_probe.py [--steps 20] [--rounds 3] [--eval-images 20]"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "denoising-vit_b200"))
sys.path.insert(0, ROOT)

import dvt.models as DVT  # noqa: E402
from dvt.dense_eval import depth_ops as O  # noqa: E402
from dvt.dense_eval.depth import DepthHead, depth_losses, metrics_from_sums  # noqa: E402
from dvt.dense_eval.model import ProbeBackbone  # noqa: E402
from oracle import depth as OD  # noqa: E402

IDENT = "vit_base_patch14_dinov2.lvd142m"


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return q


def torch_step(head, feat, cls, gt):
    """The reference's order in torch (float32): upsample cat(feat, cls) x4, conv, ..., resize, losses."""
    d4 = OD.head_forward(feat.permute(0, 3, 1, 2), cls, head.conv_depth.weight, head.conv_depth.bias, head.bins, 4)
    ld, lg, tot = OD.loss(d4, gt[:, None], warm_up=False)
    return tot


def ours_step(head, feat, cls, gt, sig):
    return depth_losses(head(feat, cls), gt, sig, 1.0, 0.5)["loss"]


def time_train(backbone, B, steps, rounds):
    g = torch.Generator(device="cuda").manual_seed(B)
    img = torch.randn(B, 3, 416, 544, device="cuda", generator=g)
    gt = torch.rand(B, 416, 544, device="cuda", generator=g) * 9 + 0.5
    torch.manual_seed(0)
    head = DepthHead(1536, 256, 0.001, 10, 4).cuda()
    opt = torch.optim.AdamW(head.parameters(), lr=1e-4)
    sig = O.SigLossState(warm_up=False)
    feat, cls = backbone(img)
    arms = {"sm90a": lambda: ours_step(head, feat, cls, gt, sig), "torch_ref": lambda: torch_step(head, feat, cls, gt)}
    loss0 = {k: f().item() for k, f in arms.items()}
    res = {k: [] for k in arms}
    peak = {}
    for _ in range(rounds):
        for name, f in arms.items():
            for _ in range(3):  # warm-up
                opt.zero_grad(set_to_none=True)
                f().backward()
            torch.cuda.synchronize()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            for _ in range(steps):
                feat, cls = backbone(img)          # the frozen forward is part of a step
                opt.zero_grad(set_to_none=True)
                arms[name]().backward()
                opt.step()
            torch.cuda.synchronize()
            res[name].append((time.perf_counter() - t0) * 1e3 / steps)
            peak[name] = torch.cuda.max_memory_allocated() / 2 ** 20
    out = {}
    for name, ts in res.items():
        ts = sorted(ts)
        out[name] = {"step_ms_median": round(ts[len(ts) // 2], 3), "step_ms_range": [round(ts[0], 3), round(ts[-1], 3)],
                     "peak_mib": round(peak[name], 1)}
    out["loss_span"] = abs(loss0["sm90a"] - loss0["torch_ref"])
    return out


def time_eval(backbone, n_images):
    torch.manual_seed(0)
    head = DepthHead(1536, 256, 0.001, 10, 4).cuda().eval()
    g = torch.Generator(device="cuda").manual_seed(1)
    img = torch.randn(1, 3, 480, 640, device="cuda", generator=g)
    gt = torch.rand(480, 640, device="cuda", generator=g) * 11
    ws = torch.empty(O.EVAL_WORKSPACE, dtype=torch.float64, device="cuda")
    sums = torch.zeros(10, dtype=torch.float64, device="cuda")
    crop = (45, 471, 41, 601)

    @torch.no_grad()
    def ours():
        x = torch.cat([img, img.flip(3)])
        O.eval_sums(head(*backbone(x)), [False, True], gt, 0.001, 10, crop, sums, ws)
        return metrics_from_sums(sums.cpu().numpy())

    @torch.no_grad()
    def ref():
        x = torch.cat([img, img.flip(3)])
        feat, cls = backbone(x)
        d4 = OD.head_forward(feat.permute(0, 3, 1, 2), cls, head.conv_depth.weight, head.conv_depth.bias, head.bins, 4)
        pred = OD.aug_predict(d4, [False, True], gt.shape, 0.001, 10)
        m = OD.eval_mask(gt.cpu().numpy(), 0.001, 10, crop)
        return OD.calculate(gt.cpu().numpy()[m].astype("float64"), pred.cpu().numpy()[m].astype("float64"))

    out = {}
    for name, f in (("sm90a", ours), ("torch_ref", ref)):
        f()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n_images):
            vals = f()
        torch.cuda.synchronize()
        out[name] = {"images_per_s": round(n_images / (time.perf_counter() - t0), 2),
                     "abs_rel": float(vals[3])}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--eval-images", type=int, default=20)
    a = ap.parse_args()
    vit = DVT.PretrainedViTWrapper(IDENT, stride=14, allow_random_init=True).cuda().eval()
    backbone = ProbeBackbone(vit, [11], [0], return_cls=True, norm=True)
    res = {"card": card(), "backbone": IDENT + " (random weights)"}
    for B in (2, 8):
        res[f"train_b{B}"] = time_train(backbone, B, a.steps, a.rounds)
    res["eval_480x640_flip"] = time_eval(backbone, a.eval_images)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
