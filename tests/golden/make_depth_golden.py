"""Generates the goldens of the NYU depth probe from the reference sources:

- tests/golden/depth_losses.npz: SigLoss (warm-up and steady state) and GradientLoss of the reference's
  evaluation/depth/models/losses/{sigloss,gradientloss}.py, executed with a stub LOSSES registry, on seeded
  [B, 1, 12, 16] predictions and ground truths (about a fifth of the pixels invalid) for B = 1, 2, 3, 5, and on an
  all-invalid ground truth;
- tests/golden/depth_metrics.npz: calculate() of evaluation/depth/core/evaluation/metrics.py (mmcv stubbed: the module
  only imports it) on seeded float32 gt / pred vectors, an empty one included;
- tests/golden/depth_config.json: the top-level names of evaluation/configs/vitb_nyu_linear_config.py as executed by
  Python, in JSON form (tuples as lists).

Run in the build container (needs /root/reference):  python tests/golden/make_depth_golden.py"""
import json
import os
import runpy
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"


class _Registry:
    def register_module(self, *a, **k):
        return lambda cls: cls


def _load(path, package_stubs):
    src = open(path).read()
    for old, new in package_stubs:
        src = src.replace(old, new)
    ns = {"__name__": "ref_" + os.path.basename(path)[:-3], "LOSSES": _Registry()}
    exec(compile(src, path, "exec"), ns)
    return ns


def jsonable(v):
    if isinstance(v, dict):
        return {k: jsonable(x) for k, x in v.items()}
    if isinstance(v, (list, tuple, range)):
        return [jsonable(x) for x in v]
    return v


if __name__ == "__main__":
    losses = os.path.join(REF, "evaluation", "depth", "models", "losses")
    stub = [("from ...models.builder import LOSSES", "")]
    SigLoss = _load(os.path.join(losses, "sigloss.py"), stub)["SigLoss"]
    GradientLoss = _load(os.path.join(losses, "gradientloss.py"), stub)["GradientLoss"]
    sys.modules.setdefault("mmcv", types.ModuleType("mmcv"))
    calculate = _load(os.path.join(REF, "evaluation", "depth", "core", "evaluation", "metrics.py"), [])["calculate"]

    out = {}
    g = torch.Generator().manual_seed(0)
    for B in (1, 2, 3, 5):
        pred = (torch.rand(B, 1, 12, 16, generator=g, dtype=torch.float64) * 9 + 0.5)
        gt = torch.rand(B, 1, 12, 16, generator=g, dtype=torch.float64) * 9 + 0.5
        gt[torch.rand(B, 1, 12, 16, generator=g) < 0.2] = 0
        warm = SigLoss(valid_mask=True, loss_weight=1.0, warm_up=True, warm_iter=1)
        out[f"b{B}_pred"], out[f"b{B}_gt"] = pred.numpy(), gt.numpy()
        out[f"b{B}_sig_warm"] = warm(pred, gt).numpy()          # first call: warm-up branch
        out[f"b{B}_sig"] = warm(pred, gt).numpy()               # second call: steady state
        out[f"b{B}_grad"] = GradientLoss(valid_mask=True, loss_weight=0.5)(pred, gt).numpy()
    pred = torch.rand(2, 1, 12, 16, generator=g, dtype=torch.float64) + 1
    zero = torch.zeros_like(pred)
    out["invalid_pred"] = pred.numpy()
    out["invalid_sig"] = SigLoss(valid_mask=True, warm_up=False)(pred, zero).numpy()
    out["invalid_grad"] = GradientLoss(valid_mask=True, loss_weight=0.5)(pred, zero).numpy()
    np.savez(os.path.join(HERE, "depth_losses.npz"), **out)

    rs = np.random.RandomState(0)
    met = {}
    for i, n in enumerate((1000, 37, 0)):
        gt = rs.uniform(0.01, 10, n).astype(np.float32)
        pred = (gt * rs.uniform(0.6, 1.5, n)).astype(np.float32)
        met[f"m{i}_gt"], met[f"m{i}_pred"] = gt, pred
        met[f"m{i}_out"] = np.array(calculate(gt, pred), dtype=np.float64)
    np.savez(os.path.join(HERE, "depth_metrics.npz"), **met)

    ns = runpy.run_path(os.path.join(REF, "evaluation", "configs", "vitb_nyu_linear_config.py"))
    with open(os.path.join(HERE, "depth_config.json"), "w") as fh:
        json.dump(jsonable({k: v for k, v in ns.items() if not k.startswith("__")}), fh, indent=1, sort_keys=True)
    print(sorted(out), sorted(met))
