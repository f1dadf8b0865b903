#!/usr/bin/env python
"""Throughput of the DINOv3 ViT-B/16 backbone (2-D RoPE fused into the QKV GEMM epilogue).

  * extraction images/s (stage 1, `--extract-bsz` views per forward) at 224 x 224 stride 16 and at 512 x 512 stride 8;
  * one stage-3 step (forward, loss, backward, gradient checkpointing) at 512 x 512 stride 16;
  * the QKV GEMM of ViT-B at the two extraction shapes, with the RoPE epilogue (dvt_gemm_qkv_rope) and without it
    (dvt_gemm_tn with the bias-only epilogue, the DINOv2 form), timed alternately in the same run.

GPU only.  CUDA-event timing after warm-up (tools/bench_backbones.py helpers); the GPU name and power limit are read in the
same run.  One JSON line.  Writes nothing to the tree.

  python tools/bench_dinov3.py [--steps 10 --warmup 3]"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "denoising-vit_b200"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)

from bench_backbones import _gpu_info, _time, extraction, stage3_step  # noqa: E402

BASE = "vit_base_patch16_dinov3.lvd1689m"


def qkv_gemm(batch, size, stride, steps, warmup, rounds=3):
    from dvt import ops, train_ops
    from dvt.models import vit_wrapper as VW
    C, prefix = 768, 5
    h = w = (size - 16) // stride + 1
    ntok = prefix + h * w
    M = batch * ntok
    x = torch.randn(M, C, device="cuda").bfloat16()
    wq = (torch.randn(3 * C, C, device="cuda") / C ** 0.5).bfloat16()
    bias = torch.randn(3 * C, device="cuda")
    rope = VW.rope_table(h, w).cuda()
    plain = lambda: ops.gemm_tn(x, wq, bias, None, torch.bfloat16)                      # noqa: E731
    fused = lambda: train_ops.gemm_qkv_rope(x, wq, bias, rope, batch, prefix, C // 64)  # noqa: E731
    t_plain, t_rope = [], []
    for _ in range(rounds):                    # alternate the two forms: other work shares the host
        t_plain.append(_time(plain, steps, warmup))
        t_rope.append(_time(fused, steps, warmup))
    fl = 2.0 * M * 3 * C * C
    tp, tr = min(t_plain), min(t_rope)
    return {"M": M, "N": 3 * C, "K": C, "plain_ms": round(tp * 1e3, 4), "rope_ms": round(tr * 1e3, 4),
            "plain_tflops": round(fl / tp / 1e12, 1), "rope_tflops": round(fl / tr / 1e12, 1),
            "rope_over_plain": round(tr / tp, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--extract-bsz", type=int, default=16, help="views per extraction batch (stage 1)")
    ap.add_argument("--stage3-batch", type=int, default=4)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "GPU only"
    res = {"gpu": _gpu_info(), "extraction": [], "stage3": None, "qkv_gemm": []}
    res["extraction"].append(extraction(BASE, 224, 16, a.extract_bsz, a.steps, a.warmup))
    res["extraction"].append(extraction(BASE, 512, 8, max(1, a.extract_bsz // 4), max(2, a.steps // 2), 1))
    res["stage3"] = stage3_step(BASE, 512, 16, a.stage3_batch, max(2, a.steps // 2), 1)
    res["qkv_gemm"].append(qkv_gemm(a.extract_bsz, 224, 16, 4 * a.steps, a.warmup))
    res["qkv_gemm"].append(qkv_gemm(max(1, a.extract_bsz // 4), 512, 8, 2 * a.steps, a.warmup))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
