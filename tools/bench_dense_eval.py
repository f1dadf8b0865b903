"""Measures the segmentation probe on one GPU: ViT-B/14 DINOv2 layout (random weights), synthetic inputs.

1. Training step on 512 x 512 crops (batch 2 and 8, K = 21 and 150): `step_ms` is the host wall-clock time per plain
   step (forward, `loss.backward()`, AdamW) over `--iters` back-to-back steps with no synchronisation inside the window,
   with the peak memory of those steps.  The `*_span_ms` fields come from a second loop that splits the same step at
   the phase boundaries (the backward in two calls: to the logits, then through the head) and records CUDA events:
   backbone forward, head (BN + 1x1 conv, forward and backward), loss (upsample + cross-entropy, forward and backward
   to the low-resolution logits) and AdamW.  They are spans on the device timeline and include any time the GPU waits
   for the host to launch that phase's kernels, so they need not add up to `step_ms`.  The fused kernel (`dvt_seg_upsample_ce`) is
   measured beside the torch statement (`F.interpolate` + `F.cross_entropy`) under the same backbone and head, the two
   alternating, `--repeats` rounds.
2. Slide inference (crop 512, stride 341, test-time keep-ratio resize into (2048, 512)) of 500 x 375 and 2048 x 512
   images, K = 21 and 150: images/s through the two inference kernels beside a torch restatement of mmseg's
   slide_inference (F.interpolate, F.pad, division, resize, argmax, bincount histograms).

Prints the card name and power limit, then one JSON line per measurement.
Usage: python tools/bench_dense_eval.py [--iters 20] [--warmup 5] [--repeats 3]"""
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

import dvt.models as DVT  # noqa: E402
from dvt.dense_eval import seg_ops  # noqa: E402
from dvt.dense_eval.data import rescale_size, slide_windows  # noqa: E402
from dvt.dense_eval.model import LinearSegHead, ProbeBackbone  # noqa: E402

IDENT = "vit_base_patch14_dinov2.lvd142m"


def torch_loss(logits_nhwc, labels):
    up = F.interpolate(logits_nhwc.permute(0, 3, 1, 2), size=labels.shape[1:], mode="bilinear", align_corners=False)
    return F.cross_entropy(up, labels.long(), reduction="none", ignore_index=255).mean()


def bench_train(backbone, B, K, fused, iters, warmup):
    head = LinearSegHead(768, K).cuda()
    opt = torch.optim.AdamW(head.parameters(), lr=1e-3, betas=(0.9, 0.999), weight_decay=1e-4)
    g = torch.Generator().manual_seed(0)
    img = torch.randn(B, 3, 512, 512, generator=g).cuda()
    seg = torch.randint(0, K, (B, 512, 512), generator=g).to(torch.uint8)
    seg[:, 400:] = 255
    seg = seg.cuda()
    lossfn = seg_ops.upsample_cross_entropy if fused else torch_loss
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    for i in range(warmup + iters):          # the plain training step, timed by the host clock
        if i == warmup:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
        loss = lossfn(head(backbone(img)), seg)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) / iters * 1e3
    peak = torch.cuda.max_memory_allocated() / 1e9
    parts = {"backbone": 0.0, "head": 0.0, "loss": 0.0, "optimizer": 0.0}
    timed = []
    for i in range(warmup + iters):          # the same step split at the phase boundaries, spans from CUDA events
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
        ev[0].record()
        feats = backbone(img)
        ev[1].record()
        logits = head(feats)
        ev[2].record()
        loss = lossfn(logits, seg)
        (dl,) = torch.autograd.grad(loss, logits)
        ev[3].record()
        opt.zero_grad(set_to_none=True)
        logits.backward(dl)
        ev[4].record()
        opt.step()
        ev[5].record()
        if i >= warmup:
            timed.append(ev)
    torch.cuda.synchronize()
    for ev in timed:
        for k, (a, b) in zip(("backbone", "loss", "optimizer"), ((0, 1), (2, 3), (4, 5))):
            parts[k] += ev[a].elapsed_time(ev[b]) / iters
        parts["head"] += (ev[1].elapsed_time(ev[2]) + ev[3].elapsed_time(ev[4])) / iters
    return dict(kind="train_step", path="fused" if fused else "torch", batch=B, K=K, step_ms=round(wall, 3),
                **{f"{k}_span_ms": round(v, 3) for k, v in parts.items()},
                peak_mem_gb=round(peak, 3))


def torch_slide_hist(logits_fn, img, gt, K, crop, stride, hist):
    H, W = img.shape[1:]
    wins = slide_windows(H, W, crop, stride)
    preds = torch.zeros(1, K, H, W, device=img.device)
    count = torch.zeros(1, 1, H, W, device=img.device)
    crops = torch.stack([img[:, y1:y2, x1:x2] for (y1, y2, x1, x2) in wins])
    logits = logits_fn(crops).permute(0, 3, 1, 2)
    for j, (y1, y2, x1, x2) in enumerate(wins):
        cl = F.interpolate(logits[j:j + 1], size=(y2 - y1, x2 - x1), mode="bilinear", align_corners=False)
        preds += F.pad(cl, (x1, W - x2, y1, H - y2))
        count[:, :, y1:y2, x1:x2] += 1
    preds = F.interpolate(preds / count, size=gt.shape, mode="bilinear", align_corners=False)
    pred = preds.argmax(1)[0]
    m = gt != 255
    p, t = pred[m], gt[m].long()
    inter = torch.bincount(p[p == t], minlength=K)
    ap, al = torch.bincount(p, minlength=K), torch.bincount(t[t < K], minlength=K)
    hist += torch.stack([inter, ap + al - inter, ap, al])


@torch.no_grad()
def bench_slide(backbone, K, orig_hw, fused, iters, warmup):
    head = LinearSegHead(768, K).cuda().eval()
    fn = lambda crops: head(backbone(crops))  # noqa: E731
    Ho, Wo = orig_hw
    h, w = rescale_size(Ho, Wo, (2048, 512))
    g = torch.Generator().manual_seed(1)
    img = torch.randn(3, h, w, generator=g).cuda()
    gt = torch.randint(0, K, (Ho, Wo), generator=g).to(torch.uint8).cuda()
    hist = torch.zeros(4, K, dtype=torch.int64, device="cuda")
    run = (lambda: seg_ops.slide_inference_hist(fn, img, gt, K, (512, 512), (341, 341), hist)) if fused else \
        (lambda: torch_slide_hist(fn, img, gt, K, (512, 512), (341, 341), hist))
    for _ in range(warmup):
        run()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        run()
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / iters
    return dict(kind="slide_inference", path="fused" if fused else "torch", K=K, image=f"{Wo}x{Ho}", resized=f"{w}x{h}",
                windows=len(slide_windows(h, w, (512, 512), (341, 341))), ms_per_image=round(ms, 3),
                images_per_s=round(1000.0 / ms, 2), peak_mem_gb=round(torch.cuda.max_memory_allocated() / 1e9, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_dense_eval needs a GPU"
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        smi = "nvidia-smi unavailable"
    print(json.dumps({"device": torch.cuda.get_device_name(0), "nvidia_smi": smi}), flush=True)
    torch.manual_seed(0)
    vit = DVT.PretrainedViTWrapper(IDENT, stride=14, allow_random_init=True).cuda().eval()
    for p in vit.parameters():
        p.requires_grad = False
    backbone = ProbeBackbone(vit, [8, 9, 10, 11], [3])
    for rep in range(args.repeats):
        for B in (2, 8):
            for K in (21, 150):
                for fused in ((True, False) if rep % 2 == 0 else (False, True)):
                    r = bench_train(backbone, B, K, fused, args.iters, args.warmup)
                    print(json.dumps(dict(r, repeat=rep)), flush=True)
    for K in (21, 150):
        for hw in ((375, 500), (512, 2048)):
            for fused in (True, False):
                print(json.dumps(bench_slide(backbone, K, hw, fused, args.iters, args.warmup)), flush=True)


if __name__ == "__main__":
    main()
