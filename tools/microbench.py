#!/usr/bin/env python
"""Per-kernel timings at the headline shapes (ViT-B/14, 518^2, batch B views; fit with C=768, 2048 pixels, 16 levels).
CUDA events around back-to-back launches after warm-up, L2 flushed between timed launches unless --no-flush."""
import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "denoising-vit_b200"))
from dvt import ops  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--only", type=str, default="")
    ap.add_argument("--no-flush", action="store_true")
    a = ap.parse_args()
    dev = "cuda"
    B, N, C, H = a.batch, 1370, 768, 12
    M = B * N
    g = torch.Generator(device=dev).manual_seed(0)
    rn = lambda *s: torch.randn(*s, device=dev, generator=g)  # noqa: E731
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)

    x = rn(M, C)
    xn = rn(M, C).bfloat16()
    w_qkv, b_qkv = (rn(3 * C, C) / 28).bfloat16(), rn(3 * C)
    w_proj, b_proj = (rn(C, C) / 28).bfloat16(), rn(C)
    w_fc1, b_fc1 = (rn(4 * C, C) / 28).bfloat16(), rn(4 * C)
    w_fc2, b_fc2 = (rn(C, 4 * C) / 55).bfloat16(), rn(C)
    hid = rn(M, 4 * C).bfloat16()
    qkv = rn(B, N, 3 * C).bfloat16()
    gam = torch.ones(C, device=dev)
    lnw, lnb = torch.ones(C, device=dev), torch.zeros(C, device=dev)
    img = rn(B, 3, 518, 518)
    cols = ops.im2col(img, 14, 14)
    w_pe = (rn(C, cols.shape[1]) / 24).bfloat16()

    cases = {
        "layernorm": (lambda: ops.layernorm(x, lnw, lnb), 0, M * C * 6),
        "gemm_qkv": (lambda: ops.gemm_tn(xn, w_qkv, b_qkv, None, torch.bfloat16), 2 * M * 3 * C * C, 0),
        "attention": (lambda: ops.attention(qkv, H), 4 * B * H * N * N * 64, 0),
        "gemm_proj_resid": (lambda: ops.gemm_tn_residual_(x, xn, w_proj, b_proj, gam), 2 * M * C * C, 0),
        "gemm_fc1_gelu": (lambda: ops.gemm_tn(xn, w_fc1, b_fc1, "gelu", torch.bfloat16), 2 * M * 4 * C * C, 0),
        "gemm_fc2_resid": (lambda: ops.gemm_tn_residual_(x, hid, w_fc2, b_fc2, gam), 2 * M * 4 * C * C, 0),
        "im2col": (lambda: ops.im2col(img, 14, 14), 0, B * 1369 * 592 * 2 + B * 3 * 518 * 518 * 4),
        "gemm_patch": (lambda: ops.gemm_tn(cols, w_pe, b_proj, None, torch.float32), 2 * B * 1369 * C * 588, 0),
    }
    print(f"{'kernel':<18}{'ms':>9}{'TFLOP/s':>10}{'GB/s':>9}   (batch {B}, M={M})")
    for name, (fn, flops, byts) in cases.items():
        if a.only and a.only != name:
            continue
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(a.iters):
            if not a.no_flush:
                flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ms = float(np.median(ts))
        print(f"{name:<18}{ms:>9.3f}{flops / ms / 1e9 if flops else 0:>10.1f}{byts / ms / 1e6 if byts else 0:>9.0f}")


if __name__ == "__main__":
    main()
