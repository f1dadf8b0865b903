"""Mints tests/golden/fit_headline_2000.npz: a FULL-LENGTH fit at the headline size, run by the REFERENCE's own classes.

SURVEY.md section 8(c) asks for a 2000-step trajectory at the size BASELINE.json's metric is quoted on: feat_dim 768,
37 x 37 noise map, 16 hash-grid levels (the last one hashed, 19 741 760 table parameters), 2048 sampled pixels per
step, loss scale 1024, warm-up pinned to 200, G frozen / residual MLP started after step 1000.  Only the number of
views is small (V = 3, so the bank fits a fixture-free, seed-derived tensor and the CPU run takes minutes, not hours).

Like make_fit_golden.py it drives `dvt/models/offline_denoiser.py::SingleImageDenoiser`, `torch.optim.Adam` and
`dvt/utils/misc.py::adjust_learning_rate`, imported unmodified from /root/reference, through the loop of
main_img_denoising.py:39-89,121-130 (tiny-cuda-nn's encoding replaced by oracle/hashgrid.py).  Inputs are re-derived
from seeds by the test (`oracle.fit.synthetic_bank / init_params`, `np.random.RandomState`); only outputs are stored:
the five loss terms every 50 steps and the final `denoised_feats` (fp16: 1 - cos of the rounding is < 1e-7).

Run once, in the build container:  python tests/golden/make_fit_golden_headline.py      (~15-25 min on 8 cores)
"""
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import make_fit_golden as MG  # noqa: E402
from oracle import fit as OF  # noqa: E402
from oracle import hashgrid as HG  # noqa: E402

CFG = dict(C=768, h=37, w=37, V=3, bsz=2048, n_levels=16, num_iters=2000, warmup_iters=200, lr=0.01, min_lr=0.001,
           weight_decay=1e-5, freeze_after=0.5, loss_scale=1024.0, log_every=50, seed=7)


def inputs(cfg):
    meta = HG.grid_meta(cfg["n_levels"])
    feats, coords = OF.synthetic_bank(cfg["V"], cfg["h"], cfg["w"], cfg["C"], seed=cfg["seed"])
    init = OF.init_params(cfg["C"], cfg["h"], cfg["w"], meta, seed=cfg["seed"])
    idx = np.random.RandomState(cfg["seed"]).randint(0, cfg["V"] * cfg["h"] * cfg["w"], (cfg["num_iters"], cfg["bsz"]))
    return meta, feats, coords, init, idx


if __name__ == "__main__":
    torch.set_num_threads(int(os.environ.get("DVT_GOLDEN_THREADS", os.cpu_count())))
    cfg = dict(CFG)
    if len(sys.argv) > 1:
        cfg["num_iters"] = int(sys.argv[1])  # (smoke run of the script itself)
    meta, feats, coords, init, idx = inputs(cfg)
    t0 = time.time()
    ref = MG.reference_run(cfg, feats, coords, meta, init, idx)
    print(f"reference run: {cfg['num_iters']} steps in {time.time() - t0:.0f} s; final loss {ref['logs'][-1][1]:.5f}")
    arrays = {"cfg_keys": np.array(sorted(cfg)), "cfg_vals": np.array([float(cfg[k]) for k in sorted(cfg)]),
              "logs": ref["logs"], "denoised_feats": ref["denoised_feats"].numpy().astype(np.float16),
              "idx_checksum": np.array([int(idx.sum())]),
              "table_sum": np.array([float(ref["table"].double().sum()), float(ref["table"].double().abs().sum())])}
    name = "fit_headline_2000.npz" if cfg["num_iters"] == CFG["num_iters"] else f"fit_headline_{cfg['num_iters']}.npz"
    path = os.path.join(HERE, name)
    # the [1, 37, 37, 768] fp16 map is 2.1 MB: rows [0, 13) stay in the main file, [13, 26) and [26, 37) go to
    # <name>_part1.npz / _part2.npz (every file stays under 1 MB; tests/test_fit_gpu.py:_golden joins them)
    feats = arrays.pop("denoised_feats")
    bands = [(0, 13), (13, 26), (26, feats.shape[1])]
    np.savez_compressed(path, denoised_feats=feats[:, :13], **arrays)
    for i, (r0, r1) in enumerate(bands[1:], 1):
        np.savez_compressed(path.replace(".npz", f"_part{i}.npz"), denoised_feats=feats[:, r0:r1])
    print(f"wrote {path} ({os.path.getsize(path) // 1024} KiB) and its parts")
