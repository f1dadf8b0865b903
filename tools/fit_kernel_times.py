#!/usr/bin/env python
"""Per-kernel device time of the HP-2 fit at the headline size (C=768, 37x37, 2048 pixels, 16 levels) under the current
DVT_FIT_* settings: torch.profiler (CUDA activities) over a graphed fit; prints the mean time and the count per step of
the encode and table-sweep kernels (all instances of each template)."""
import argparse
import os
import sys
from collections import defaultdict

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "denoising-vit_b200"))
import dvt.models as DVT  # noqa: E402
from dvt.fit import FitEngine  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--graph-steps", type=int, default=20)
    ap.add_argument("--views", type=int, default=64)
    a = ap.parse_args()
    C, h, w, V, bsz = 768, 37, 37, a.views, 2048
    field = DVT.NeuralFeatureField(feat_dim=C, n_levels=16)
    den = DVT.SingleImageDenoiser(h, w, C)
    g = torch.Generator(device="cuda").manual_seed(0)
    bank = torch.randn(V * h * w, C, device="cuda", generator=g)
    coords = torch.rand(V * h * w, 2, device="cuda", generator=g)
    idx = np.random.RandomState(0).randint(0, V * h * w, (a.iters, bsz))
    hyper = dict(lr=0.01, min_lr=0.001, warmup_iters=a.iters // 10, freeze_after=0.5, weight_decay=1e-5, loss_scale=1024.0)
    eng = FitEngine(C, h, w, bsz, field.meta)
    eng.load_modules(den, field)
    eng.begin(bank, coords, idx, **hyper)   # warm-up: graph capture, first touch
    eng.run(graph_steps=a.graph_steps)
    torch.cuda.synchronize()
    eng.begin(bank, coords, idx, **hyper)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.run(graph_steps=a.graph_steps)
        torch.cuda.synchronize()
    tot, cnt = defaultdict(float), defaultdict(int)
    for e in prof.events():
        for key in ("fit_encode_kernel", "fit_adam_table_kernel"):
            if key in e.name:
                tot[key] += e.device_time_total
                cnt[key] += 1
    for key in sorted(tot):
        print(f"{key:28s} {tot[key] / cnt[key]:8.1f} us mean  {cnt[key] / a.iters:5.2f} launches/step  "
              f"{tot[key] / a.iters:8.1f} us/step")


if __name__ == "__main__":
    main()
