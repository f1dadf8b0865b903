"""Measures multi-scale + flip evaluation of the segmentation probe on one GPU: ViT-B/14 DINOv2 layout (random weights),
synthetic inputs.

mmseg's "+ms" protocol: img_ratios 0.5, 0.75, 1.0, 1.25, 1.5, 1.75 of img_scale (2048, 512) with flip, 12
augmentations per image, slide inference (crop 512, stride 341) of each.  Original images of 683 x 512 and 2048 x 512
(ADE-like), K = 21 and 150.  The augmented images are made on the GPU before the timed region (the data pipeline runs in
DataLoader workers).  Two paths under the same backbone and head:
- "fused": `seg_ops.aug_slide_inference_hist` (windows batched 8 at a time across augmentations, the slide-window and
  test-time-augmentation kernels, histograms on the GPU);
- "torch": a torch restatement of mmseg's slide_inference + inference + aug_test (windows batched 8 at a time within an
  augmentation, where mmseg runs one; F.interpolate, F.pad, division, resize, softmax, flip, sum, argmax) with bincount
  histograms.
images/s from CUDA events over `--iters` images after `--warmup`, and the peak memory of those images; the two paths
alternate, `--repeats` rounds.  Before them, `dvt_seg_aug_accumulate` alone at the largest augmentation of each image
(CUDA events over 20 launches, with the bytes it must move per second).  Prints the card name and power limit, then one
JSON line per measurement.
Usage: python tools/bench_seg_tta.py [--iters 3] [--warmup 1] [--repeats 3]"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "denoising-vit_b200"))

import dvt.models as DVT  # noqa: E402
from dvt.dense_eval import seg_ops  # noqa: E402
from dvt.dense_eval.data import rescale_size, slide_windows  # noqa: E402
from dvt.dense_eval.model import LinearSegHead, ProbeBackbone  # noqa: E402

IDENT = "vit_base_patch14_dinov2.lvd142m"
RATIOS = [0.5, 0.75, 1.0, 1.25, 1.5, 1.75]
CROP, STRIDE, BATCH = (512, 512), (341, 341), 8


def torch_aug_test_hist(logits_fn, augs, gt, K, hist):
    seg = 0
    for img, flip in augs:
        H, W = img.shape[1:]
        wins = slide_windows(H, W, CROP, STRIDE)
        preds = torch.zeros(1, K, H, W, device=img.device)
        count = torch.zeros(1, 1, H, W, device=img.device)
        for s in range(0, len(wins), BATCH):
            chunk = wins[s:s + BATCH]
            logits = logits_fn(torch.stack([img[:, y1:y2, x1:x2] for (y1, y2, x1, x2) in chunk])).permute(0, 3, 1, 2)
            for j, (y1, y2, x1, x2) in enumerate(chunk):
                cl = F.interpolate(logits[j:j + 1], size=(y2 - y1, x2 - x1), mode="bilinear", align_corners=False)
                preds += F.pad(cl, (x1, W - x2, y1, H - y2))
                count[:, :, y1:y2, x1:x2] += 1
        out = F.softmax(F.interpolate(preds / count, size=gt.shape, mode="bilinear", align_corners=False), dim=1)
        seg = seg + (out.flip(3) if flip else out)
    pred = (seg / len(augs)).argmax(1)[0]
    m = gt != 255
    p, t = pred[m], gt[m].long()
    inter = torch.bincount(p[p == t], minlength=K)
    ap, al = torch.bincount(p, minlength=K), torch.bincount(t[t < K], minlength=K)
    hist += torch.stack([inter, ap + al - inter, ap, al])


@torch.no_grad()
def bench(fn, K, orig_hw, fused, iters, warmup):
    Ho, Wo = orig_hw
    g = torch.Generator().manual_seed(1)
    img = torch.randn(1, 3, Ho, Wo, generator=g).cuda()
    gt = torch.randint(0, K, (Ho, Wo), generator=g).to(torch.uint8).cuda()
    augs = []
    for r in RATIOS:
        a = F.interpolate(img, size=rescale_size(Ho, Wo, (int(2048 * r), int(512 * r))), mode="bilinear",
                          align_corners=False)[0]
        augs += [(a.contiguous(), False), (a.flip(2).contiguous(), True)]
    hist = torch.zeros(4, K, dtype=torch.int64, device="cuda")
    run = (lambda: seg_ops.aug_slide_inference_hist(fn, augs, gt, K, CROP, STRIDE, hist, max_batch=BATCH)) if fused else \
        (lambda: torch_aug_test_hist(fn, augs, gt, K, hist))
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
    windows = sum(len(slide_windows(x.shape[1], x.shape[2], CROP, STRIDE)) for x, _ in augs)
    return dict(kind="ms_flip_inference", path="fused" if fused else "torch", K=K, image=f"{Wo}x{Ho}", augmentations=len(augs),
                windows=windows, ms_per_image=round(ms, 2), images_per_s=round(1000.0 / ms, 3),
                peak_mem_gb=round(torch.cuda.max_memory_allocated() / 1e9, 3))


def bench_kernel(K, orig_hw, launches=20):
    """dvt_seg_aug_accumulate alone at the largest augmentation (ratio 1.75) of an image: CUDA events over `launches`
    back-to-back launches; bytes = acc and count read once, prob read and written once."""
    Ho, Wo = orig_hw
    Hc, Wc = rescale_size(Ho, Wo, (int(2048 * 1.75), int(512 * 1.75)))
    acc = torch.randn(K, Hc, Wc, device="cuda")
    count = torch.ones(Hc, Wc, device="cuda")
    prob = torch.zeros(K, Ho, Wo, device="cuda")
    seg_ops.aug_accumulate(acc, count, True, prob)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(launches):
        seg_ops.aug_accumulate(acc, count, True, prob)
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / launches
    nbytes = 4 * (K * Hc * Wc + Hc * Wc + 2 * K * Ho * Wo)
    return dict(kind="aug_accumulate_kernel", K=K, image=f"{Wo}x{Ho}", augmented=f"{Wc}x{Hc}", ms=round(ms, 3),
                gb_per_s=round(nbytes / ms / 1e6, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_seg_tta needs a GPU"
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        smi = "nvidia-smi unavailable"
    print(json.dumps({"device": torch.cuda.get_device_name(0), "nvidia_smi": smi}), flush=True)
    torch.manual_seed(0)
    vit = DVT.PretrainedViTWrapper(IDENT, stride=14, allow_random_init=True).cuda().eval()
    backbone = ProbeBackbone(vit, [8, 9, 10, 11], [3])
    for K in (21, 150):
        for hw in ((512, 683), (512, 2048)):
            print(json.dumps(bench_kernel(K, hw)), flush=True)
    for rep in range(args.repeats):
        for K in (21, 150):
            head = LinearSegHead(768, K).cuda().eval()
            fn = lambda crops: head(backbone(crops))  # noqa: E731
            for hw in ((512, 683), (512, 2048)):
                for fused in ((True, False) if rep % 2 == 0 else (False, True)):
                    print(json.dumps(dict(bench(fn, K, hw, fused, args.iters, args.warmup), repeat=rep)), flush=True)


if __name__ == "__main__":
    main()
