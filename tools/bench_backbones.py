#!/usr/bin/env python
"""Throughput of the backbones added with the head_dim-80 attention: the CLIP towers (pre_norm) and ViT-H/14 MAE.

  * extraction images/s of each backbone at the stage-1 view batch (`--extract-bsz` views per forward), at native size
    and at 518 x 518 with stride 7 (ViT-H) or 8 (CLIP; there a smaller batch);
  * flash attention forward and backward TFLOP/s at head_dim 80 against head_dim 64 at the same N and C (C = 1280:
    16 x 80 or 20 x 64 heads), and the same through F.scaled_dot_product_attention (the library bar);
  * one stage-3 step (forward, loss, backward) of ViT-H with gradient checkpointing.

GPU only.  CUDA-event timing after warm-up; the GPU name and power limit are read in the same run.  One JSON line.
Writes nothing to the tree.

  python tools/bench_backbones.py [--steps 10 --warmup 3]"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "denoising-vit_b200")):
    sys.path.insert(0, p)

CLIP224, CLIP384, HUGE = "vit_base_patch16_clip_224.openai", "vit_base_patch16_clip_384.laion2b_ft_in12k_in1k", \
    "vit_huge_patch14_224.mae"


def _gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else torch.cuda.get_device_name()
    except Exception:
        return torch.cuda.get_device_name()


def _time(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps / 1e3   # seconds per call


def extraction(tag, size, stride, batch, steps, warmup):
    import dvt.models as DVT
    w = DVT.PretrainedViTWrapper(tag, stride=stride, allow_random_init=True).cuda().eval()
    x = torch.randn(batch, 3, size, size, device="cuda")
    layer = w.last_layer_index
    out = torch.empty((batch,) + tuple(w.model.patch_embed.dynamic_feat_size((size, size))) + (w.n_output_dims,),
                      device="cuda")
    with torch.no_grad():
        t = _time(lambda: w.extract_into(x, layer, out), steps, warmup)
    del w
    torch.cuda.empty_cache()
    return {"tag": tag, "size": size, "stride": stride, "batch": batch, "images_per_s": round(batch / t, 2)}


def attention(N, C, D, B, steps, warmup):
    from dvt import ops, train_ops
    H = C // D
    qkv = (torch.randn(B, N, 3 * C, device="cuda") * 1.5).bfloat16()
    dout = torch.randn(B, N, C, device="cuda").bfloat16()
    fl_f = 4.0 * B * H * N * N * D                 # QK^T and PV
    fl_b = 2.5 * fl_f                              # S and dP recomputed, dV, dK, dQ
    t_f = _time(lambda: ops.attention(qkv, H, head_dim=D), steps, warmup)
    out, lse = train_ops.attention_fwd_lse(qkv, H, head_dim=D)
    t_b = _time(lambda: train_ops.attention_bwd(qkv, out, dout, lse, H, head_dim=D), steps, warmup)
    q, k, v = qkv.view(B, N, 3, H, D).permute(2, 0, 3, 1, 4)
    q, k, v = (t.contiguous().requires_grad_(True) for t in (q, k, v))
    do = dout.view(B, N, H, D).transpose(1, 2).contiguous()
    t_sf = _time(lambda: F.scaled_dot_product_attention(q, k, v), steps, warmup)
    o = F.scaled_dot_product_attention(q, k, v)
    t_sb = _time(lambda: torch.autograd.grad(o, (q, k, v), do, retain_graph=True), steps, warmup)
    r = lambda fl, t: round(fl / t / 1e12, 1)   # noqa: E731
    return {"N": N, "C": C, "head_dim": D, "B": B, "fwd_tflops": r(fl_f, t_f), "bwd_tflops": r(fl_b, t_b),
            "sdpa_fwd_tflops": r(fl_f, t_sf), "sdpa_bwd_tflops": r(fl_b, t_sb)}


def stage3_step(tag, size, stride, batch, steps, warmup):
    import dvt.models as DVT
    from dvt import train_ops
    w = DVT.PretrainedViTWrapper(tag, stride=stride, allow_random_init=True).cuda()
    w.set_trainable(True)
    w.model.set_grad_checkpointing(True)
    x = torch.randn(batch, 3, size, size, device="cuda")
    h, wd = w.model.patch_embed.dynamic_feat_size((size, size))
    target = torch.randn(batch, h, wd, w.n_output_dims, device="cuda")

    def step():
        for p in w.parameters():
            p.grad = None
        pred = w.get_intermediate_layers(x)[0].permute(0, 2, 3, 1)
        loss, _, _ = train_ops.denoise_loss(pred, target)
        loss.backward()

    torch.cuda.reset_peak_memory_stats()
    t = _time(step, steps, warmup)
    res = {"tag": tag, "size": size, "stride": stride, "batch": batch, "grad_checkpointing": True,
           "images_per_s": round(batch / t, 2), "peak_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}
    del w
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--extract-bsz", type=int, default=16, help="views per extraction batch (stage 1)")
    ap.add_argument("--stage3-batch", type=int, default=8)
    ap.add_argument("--stage3-size", type=int, default=224)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "GPU only"
    res = {"gpu": _gpu_info(), "extraction": [], "attention": [], "stage3": None}
    for tag, native, patch, fine in ((CLIP224, 224, 16, 8), (CLIP384, 384, 16, 8), (HUGE, 224, 14, 7)):
        res["extraction"].append(extraction(tag, native, patch, a.extract_bsz, a.steps, a.warmup))
        res["extraction"].append(extraction(tag, 518, fine, max(1, a.extract_bsz // 8), max(2, a.steps // 3), 1))
    for N, B in ((257, 32), (1370, 4), (5330, 1)):
        for D in (80, 64):
            res["attention"].append(attention(N, 1280, D, B, a.steps, a.warmup))
    res["stage3"] = stage3_step(HUGE, a.stage3_size, 14, a.stage3_batch, max(2, a.steps // 2), 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
