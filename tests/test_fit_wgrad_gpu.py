"""The stage-1 fit's weight gradients dY^T [X | 1] run on the wgmma 3xTF32 GEMM, which reads transposed hi / lo copies of
dY and X written by their producers (the GEMM epilogues, the loss, the encode and the row gather) and a ones row for the
bias gradients.  A pixel batch of 1000, not a multiple of the 128-row tile, exercises the M tail of the transposed
epilogue stores and the K tail of the weight-gradient TMA boxes at the headline size (C 768, 37 x 37, 16 levels)."""
import pytest
import torch
import torch.nn.functional as F

from test_fit_gpu import _FULL, _L, _setup

pytestmark = pytest.mark.gpu

_CFG = dict(_FULL, bsz=1000)
_MLP = ("mlp.0.weight", "mlp.0.bias", "mlp.2.weight", "mlp.2.bias")
_RES = ("res.0.weight", "res.0.bias", "res.2.weight", "res.2.bias", "res.4.weight", "res.4.bias")


def _fit(cfg, graph_steps):
    from dvt.fit import FitEngine
    feats, coords, init, idx, den, field, ometa = _setup(cfg)
    eng = FitEngine(cfg["C"], cfg["h"], cfg["w"], cfg["bsz"], field.meta)
    eng.fit(den, field, feats.reshape(-1, cfg["C"]).cuda().contiguous(), coords.reshape(-1, 2).cuda().contiguous(), idx,
            graph_steps=graph_steps, lr=cfg["lr"], min_lr=cfg["min_lr"], warmup_iters=cfg["warmup_iters"],
            freeze_after=cfg["freeze_after"], weight_decay=cfg["weight_decay"], loss_scale=cfg["loss_scale"])
    torch.cuda.synchronize()
    assert _L().device_error() == 0
    return eng, feats, coords, init, idx, ometa


def test_fit_ragged_batch_first_steps_match_oracle():
    """Six steps (three per phase) against the CPU oracle: logged losses within 1e-3 relative, and every weight and bias
    of the field and residual MLPs moves along the oracle's update."""
    from oracle import fit as OF
    cfg = dict(_CFG, num_iters=6, warmup_iters=2)
    eng, feats, coords, init, idx, ometa = _fit(cfg, graph_steps=2)
    ora = OF.fit(feats, coords, cfg["h"], cfg["w"], ometa, init, idx, lr=cfg["lr"], min_lr=cfg["min_lr"],
                 weight_decay=cfg["weight_decay"], warmup_iters=cfg["warmup_iters"], freeze_after=cfg["freeze_after"],
                 loss_scale=cfg["loss_scale"], log_every=1)
    losses = eng.losses()
    for row in ora["logs"]:
        s = int(row[0])
        for j in range(5):
            assert abs(losses[s, j] - row[1 + j]) <= 1e-3 * abs(row[1 + j]) + 1e-6, f"step {s} loss[{j}] {losses[s, j]} vs {row[1 + j]}"
    for k in _MLP + _RES:
        got = eng.get_param(k, init[k]).cpu() - init[k]
        ref = ora["params"][k] - init[k]
        moved = ref.abs() > 0
        assert moved.any(), f"{k}: the oracle does not move it"
        cos = F.cosine_similarity(got[moved].flatten().double(), ref[moved].flatten().double(), dim=0).item()
        assert cos > 0.99, f"{k}: update cosine {cos} with a pixel batch of {cfg['bsz']}"


def test_fit_ragged_batch_is_bit_exact_run_to_run():
    """Two fits of 12 steps in graphs of 4, across the phase boundary, give bit-identical parameters.  (The logged losses
    are summed over CTAs with float atomics, in arrival order: they are compared to a tolerance.)"""
    cfg = dict(_CFG, num_iters=12, warmup_iters=2)
    outs = []
    for _ in range(2):
        eng, feats, coords, init, idx, ometa = _fit(cfg, graph_steps=4)
        params = [eng.get_param(k, init[k]).cpu() for k in ("table", "G") + _MLP + _RES]
        outs.append((params, torch.from_numpy(eng.losses().copy())))
        del eng
    (pa, la), (pb, lb) = outs
    for k, a, b in zip(("table", "G") + _MLP + _RES, pa, pb):
        assert torch.equal(a, b), f"{k} differs between two identical fits (max diff {(a - b).abs().max().item()})"
    assert torch.allclose(la, lb, rtol=1e-5, atol=0), "the logged losses differ between two identical fits"
