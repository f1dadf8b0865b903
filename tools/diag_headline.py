#!/usr/bin/env python
"""Diagnoses the 2000-step headline-size fit against tests/golden/fit_headline_2000.npz under several engine settings:
per-patch cosine statistics of the final denoised_feats and the loss deviation along the trajectory."""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "denoising-vit_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
os.environ.setdefault("DVT_ALLOW_RANDOM_INIT", "1")
import test_fit_gpu as T  # noqa: E402
from dvt import _lib  # noqa: E402
from dvt.fit import FitEngine  # noqa: E402


def run(tag, env, impl=-1, graph_steps=20):
    for k in ("DVT_FIT_PIPELINE", "DVT_FIT_SWEEP_CTAS", "DVT_FIT_PDL"):
        os.environ.pop(k, None)
    os.environ.update(env)
    cfg, z = T._golden("headline_2000")
    feats, coords, init, idx, den, field, _ = T._setup(cfg)
    eng = FitEngine(cfg["C"], cfg["h"], cfg["w"], cfg["bsz"], field.meta)
    _lib.check(_lib.lib().dvt_set_debug_impl(impl))
    eng.fit(den, field, feats.reshape(-1, cfg["C"]).cuda().contiguous(), coords.reshape(-1, 2).cuda().contiguous(), idx,
            graph_steps=graph_steps, lr=cfg["lr"], min_lr=cfg["min_lr"], warmup_iters=cfg["warmup_iters"],
            freeze_after=cfg["freeze_after"], weight_decay=cfg["weight_decay"], loss_scale=cfg["loss_scale"])
    den_f = eng.query(coords[-1:].cuda()).cpu()
    torch.cuda.synchronize()
    _lib.check(_lib.lib().dvt_set_debug_impl(-1))
    ref = torch.from_numpy(z["denoised_feats"].astype(np.float32))
    cos = F.cosine_similarity(den_f.reshape(-1, cfg["C"]), ref.reshape(-1, cfg["C"]), dim=-1)
    rel = (den_f - ref).norm() / ref.norm()
    losses = eng.losses()
    dev = []
    for row in z["logs"]:
        s = int(row[0])
        dev.append((s, float(abs(losses[s, 0] - row[1]) / (abs(row[1]) + 1e-3))))
    worst = max(dev, key=lambda t: t[1])
    first_bad = next((s for s, d in dev if d > 0.02), None)
    print(f"{tag:34s} min cos {cos.min():.6f} mean {cos.mean():.6f} q01 {cos.quantile(0.01):.6f} rel-l2 {rel:.4f} | "
          f"loss dev worst {worst[1]:.4f} @ {worst[0]} first>2% @ {first_bad} | dev_err {_lib.device_error()}", flush=True)
    return den_f, losses


if __name__ == "__main__":
    a, la = run("default (pipelined, graphs 20)", {})
    b, lb = run("same again (run-to-run noise)", {})
    c, lc = run("sequential schedule", {"DVT_FIT_PIPELINE": "0"})
    d, ld = run("sequential, no graphs", {"DVT_FIT_PIPELINE": "0"}, graph_steps=0)
    cs = lambda x, y: F.cosine_similarity(x.reshape(-1, 768), y.reshape(-1, 768), dim=-1).min().item()  # noqa: E731
    print(f"run-to-run min cos {cs(a, b):.6f}; pipelined vs sequential {cs(a, c):.6f}; graphs vs none {cs(c, d):.6f}")
    if len(sys.argv) > 1 and sys.argv[1] == "simt":
        f, lf = run("sequential, SIMT fp32 GEMMs", {"DVT_FIT_PIPELINE": "0"}, impl=1, graph_steps=0)
        print(f"simt vs tensor-core sequential {cs(f, c):.6f}")
