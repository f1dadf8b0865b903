#!/usr/bin/env python
"""First steps of the headline-size fit, GPU against the CPU oracle, parameter group by parameter group: relative L2
distance of the accumulated update after T steps.  Rounding-level agreement (~1e-5) means later divergence is chaotic
amplification; a larger number points at a systematic difference."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "denoising-vit_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
os.environ.setdefault("DVT_ALLOW_RANDOM_INIT", "1")
import test_fit_gpu as T  # noqa: E402
from dvt import _lib  # noqa: E402
from dvt.fit import FitEngine  # noqa: E402
from oracle import fit as OF  # noqa: E402

KEYS = ("table", "G", "mlp.0.weight", "mlp.0.bias", "mlp.2.weight", "mlp.2.bias", "res.0.weight", "res.4.weight")

if __name__ == "__main__":
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 12
    cfg, _ = T._golden("headline_2000")
    cfg = dict(cfg, num_iters=steps, warmup_iters=max(2, steps // 4))
    if len(sys.argv) > 2:
        cfg["freeze_after"] = float(sys.argv[2])
    feats, coords, init, idx, den, field, ometa = T._setup(cfg)
    torch.set_num_threads(min(32, os.cpu_count()))
    ora = OF.fit(feats, coords, cfg["h"], cfg["w"], ometa, init, idx, lr=cfg["lr"], min_lr=cfg["min_lr"],
                 weight_decay=cfg["weight_decay"], warmup_iters=cfg["warmup_iters"], freeze_after=cfg["freeze_after"],
                 loss_scale=cfg["loss_scale"], log_every=1)
    prev = {}
    for tag, impl, env in (("tensor-core 3xTF32, sequential", 0, {"DVT_FIT_PIPELINE": "0"}), ("tensor-core 3xTF32, sequential (again)", 0, {"DVT_FIT_PIPELINE": "0"}),
                           ("SIMT fp32, sequential", 1, {"DVT_FIT_PIPELINE": "0"}), ("tensor-core 3xTF32, pipelined", 0, {})):
        os.environ.pop("DVT_FIT_PIPELINE", None)
        os.environ.update(env)
        feats, coords, init, idx, den, field, _ = T._setup(cfg)
        eng = FitEngine(cfg["C"], cfg["h"], cfg["w"], cfg["bsz"], field.meta)
        _lib.check(_lib.lib().dvt_set_debug_impl(impl))
        eng.fit(den, field, feats.reshape(-1, cfg["C"]).cuda().contiguous(), coords.reshape(-1, 2).cuda().contiguous(), idx,
                graph_steps=0, lr=cfg["lr"], min_lr=cfg["min_lr"], warmup_iters=cfg["warmup_iters"],
                freeze_after=cfg["freeze_after"], weight_decay=cfg["weight_decay"], loss_scale=cfg["loss_scale"])
        torch.cuda.synchronize()
        _lib.check(_lib.lib().dvt_set_debug_impl(-1))
        losses = eng.losses()
        ldev = max(abs(losses[int(r[0]), 0] - r[1]) / abs(r[1]) for r in ora["logs"])
        parts = []
        for k in KEYS:
            got = eng.get_param(k, init[k]).cpu().double() - init[k].double()
            ref = ora["params"][k].double() - init[k].double()
            if ref.norm() == 0:
                continue
            parts.append(f"{k} {float((got - ref).norm() / ref.norm()):.2e}")
            if os.environ.get("DIAG_ELEMENTWISE") and k in ("G", "mlp.0.weight", "mlp.2.weight", "table"):
                nz = ref.abs() > 0
                rel = ((got - ref).abs()[nz] / ref.abs()[nz])
                q = torch.quantile(rel[torch.randperm(rel.numel())[:2000000]].float(), torch.tensor([0.5, 0.9, 0.99, 0.999]))
                parts.append(f"[{k} elementwise rel: median {q[0]:.1e} p90 {q[1]:.1e} p99 {q[2]:.1e} p99.9 {q[3]:.1e} "
                             f"frac>1e-3 {float((rel > 1e-3).float().mean()):.2e} frac>0.5 {float((rel > 0.5).float().mean()):.2e}]")
            if k == "table":
                touched = ref.abs() > 1.5 * ref.abs().median()
                if touched.any():
                    parts.append(f"table(touched) {float((got - ref)[touched].norm() / ref[touched].norm()):.2e}")
        print(f"{tag:30s} T={steps} max rel loss dev {ldev:.2e} | " + "  ".join(parts), flush=True)
        cur = {k: eng.get_param(k, init[k]).cpu().double() - init[k].double() for k in KEYS}
        if prev:
            print("      vs previous GPU run: " + "  ".join(f"{k} {float((cur[k] - prev[k]).norm() / (prev[k].norm() + 1e-30)):.2e}" for k in KEYS), flush=True)
        prev = cur
