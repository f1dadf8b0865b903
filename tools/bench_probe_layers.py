"""Measures the four-layer linear probes on one GPU: the last four layers of ViT-B/14 and ViT-L/14 (DINOv2 layout, random
weights, synthetic inputs) from one pass over the blocks against one pass per layer.

Two arms under the same backbone, head and inputs:
- "one_pass": `ProbeBackbone` as it runs, `forward_layers_concat` (dvt_vit_forward_layers: the blocks once, the four maps
  written side by side in channels);
- "per_layer": one `dvt_vit_forward` per layer and torch.cat of the maps (what `ProbeBackbone` did before), 9 + 10 + 11 +
  12 = 42 block passes instead of 12 for ViT-B (90 instead of 24 for ViT-L).
Three workloads per backbone:
- "extract": the features of a batch of 8 crops of 512 x 512 (padded to 518 x 518, a 37 x 37 grid);
- "train_step": one step of the segmentation probe (batch 8, 512 x 512 crops, K = 21): features, BNHead, upsample +
  cross-entropy, backward, AdamW;
- "ms_flip_eval": multi-scale + flip slide evaluation (12 augmentations, crop 512, stride 341, K = 150) of one 2048 x 512
  image.
ms per call from CUDA events over `--iters` calls after `--warmup`; the arms alternate within each of `--repeats` rounds
(the first arm swaps every round), so the spread over rounds is the run-to-run noise.  The outputs of the two arms are
compared bit for bit first.  Prints the card name and power limit, one JSON line per measurement, then a summary line per
workload (median over rounds, min-max, ratio of medians).
Usage: python tools/bench_probe_layers.py [--iters 5] [--warmup 2] [--repeats 5] [--models base,large]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "denoising-vit_b200"))

import dvt.models as DVT  # noqa: E402
from dvt.dense_eval import seg_ops  # noqa: E402
from dvt.dense_eval.data import rescale_size  # noqa: E402
from dvt.dense_eval.model import LinearSegHead, ProbeBackbone  # noqa: E402

MODELS = {"base": "vit_base_patch14_dinov2.lvd142m", "large": "vit_large_patch14_dinov2.lvd142m"}
RATIOS = [0.5, 0.75, 1.0, 1.25, 1.5, 1.75]
CROP, STRIDE, BATCH = (512, 512), (341, 341), 8


def per_layer(probe):
    """The maps of probe.layers the way ProbeBackbone computed them before one pass served them all."""
    def fn(x):
        x = probe.pad(x)
        return torch.cat([probe.model.model._run(x, l, False, all_tokens=False) for l in probe.layers], -1)
    return fn


def timed(run, iters, warmup):
    for _ in range(warmup):
        run()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        run()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def workloads(probe, C):
    """name -> {arm: zero-argument callable}."""
    g = torch.Generator().manual_seed(0)
    crops = torch.randn(8, 3, 512, 512, generator=g).cuda()
    labels = torch.randint(0, 21, (8, 512, 512), generator=g).to(torch.uint8).cuda()
    img = torch.randn(1, 3, 512, 2048, generator=g).cuda()
    gt = torch.randint(0, 150, (512, 2048), generator=g).to(torch.uint8).cuda()
    augs = []
    for r in RATIOS:
        a = F.interpolate(img, size=rescale_size(512, 2048, (int(2048 * r), int(512 * r))), mode="bilinear",
                          align_corners=False)[0]
        augs += [(a.contiguous(), False), (a.flip(2).contiguous(), True)]
    feats = {"one_pass": probe, "per_layer": per_layer(probe)}
    out = {"extract": {}, "train_step": {}, "ms_flip_eval": {}}
    for arm, fx in feats.items():
        out["extract"][arm] = (lambda fx=fx: fx(crops))
        head = LinearSegHead(4 * C, 21).cuda().train()
        opt = torch.optim.AdamW(head.parameters(), lr=1e-3)

        def step(fx=fx, head=head, opt=opt):
            with torch.no_grad():
                f = fx(crops)
            loss = seg_ops.upsample_cross_entropy(head(f), labels)
            opt.zero_grad(set_to_none=True)
            loss.backward()
            opt.step()
        out["train_step"][arm] = step
        ev_head = LinearSegHead(4 * C, 150).cuda().eval()
        hist = torch.zeros(4, 150, dtype=torch.int64, device="cuda")

        def evaluate(fx=fx, ev_head=ev_head, hist=hist):
            with torch.no_grad():
                seg_ops.aug_slide_inference_hist(lambda c: ev_head(fx(c)), augs, gt, 150, CROP, STRIDE, hist,
                                                 max_batch=BATCH)
        out["ms_flip_eval"][arm] = evaluate
    return out, crops


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--models", default="base,large")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_probe_layers needs a GPU"
    try:
        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        smi = "nvidia-smi unavailable"
    print(json.dumps({"device": torch.cuda.get_device_name(0), "nvidia_smi": smi}), flush=True)
    for key in args.models.split(","):
        ident = MODELS[key]
        torch.manual_seed(0)
        vit = DVT.PretrainedViTWrapper(ident, stride=14, allow_random_init=True).cuda().eval()
        depth, C = vit.num_blocks, vit.n_output_dims
        layers = list(range(depth - 4, depth))
        probe = ProbeBackbone(vit, layers, [0, 1, 2, 3])
        loads, crops = workloads(probe, C)
        with torch.no_grad():
            same = torch.equal(probe(crops), per_layer(probe)(crops))
        print(json.dumps({"model": ident, "layers": layers, "outputs_bit_identical": same}), flush=True)
        times = {w: {arm: [] for arm in arms} for w, arms in loads.items()}
        for rep in range(args.repeats):
            for w, arms in loads.items():
                order = list(arms) if rep % 2 == 0 else list(arms)[::-1]
                for arm in order:
                    ms = timed(arms[arm], args.iters, args.warmup)
                    times[w][arm].append(ms)
                    print(json.dumps({"model": ident, "workload": w, "arm": arm, "repeat": rep, "ms": round(ms, 3)}),
                          flush=True)
        for w, arms in times.items():
            med = {arm: statistics.median(v) for arm, v in arms.items()}
            print(json.dumps({"summary": ident, "workload": w,
                              **{f"{arm}_ms_median": round(m, 2) for arm, m in med.items()},
                              **{f"{arm}_ms_range": [round(min(v), 2), round(max(v), 2)] for arm, v in arms.items()},
                              "per_layer_over_one_pass": round(med["per_layer"] / med["one_pass"], 3)}), flush=True)
        del vit, probe, loads
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
