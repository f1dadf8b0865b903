"""The fp64 one-step oracle of the stage-1 fit (tests/fit_oracle_fp64.py) against oracle/fit.py, without a GPU:
its gradients equal the fp32 autograd of `OF.denoiser_forward` within the envelope rule, the envelope bounds every
gradient, and its Adam restatement reproduces torch.optim.Adam driven the way `OF.fit` drives it (per-step lr, G dropped at
the freeze, the residual MLP joining there with a fresh step counter)."""
import numpy as np
import pytest
import torch

import fit_oracle_fp64 as FO
from oracle import fit as OF
from oracle import hashgrid as HG

HYPER = dict(lr=0.01, min_lr=0.001, warmup_iters=2, freeze_after=0.25, weight_decay=1e-5, loss_scale=1024.0)


def _problem(C=64, h=6, w=9, V=3, bsz=256, L=6, T=6, seed=3):
    meta = HG.grid_meta(L)
    feats, coords = OF.synthetic_bank(V, h, w, C, seed=seed)
    init = OF.init_params(C, h, w, meta, seed=seed)
    idx = np.random.RandomState(seed).randint(0, V * h * w, (T, bsz))
    return meta, feats.reshape(-1, C), coords.reshape(-1, 2), init, idx


def _autograd(p, feats, coords, rows, h, w, meta, phase2, loss_scale):
    """fp32 gradients of oracle/fit.py's forward (the reference semantics) at p."""
    V = feats.shape[0] // (h * w)
    q = {k: v.clone().float().requires_grad_(k != "G" or not phase2) for k, v in p.items()}
    gc = OF.make_patch_coordinates(h, w).unsqueeze(0).repeat(V, 1, 1, 1).reshape(-1, 2)
    idx = torch.as_tensor(rows)
    out = OF.denoiser_forward(q, feats[idx], coords[idx], meta, gc[idx], phase2)
    (out["loss"] * loss_scale).backward()
    return {k: v.grad for k, v in q.items() if v.grad is not None}, out


@pytest.mark.parametrize("phase2", [False, True], ids=["phase1", "phase2"])
def test_oracle_gradients_match_fp32_autograd_within_envelope(phase2):
    h, w = 6, 9
    meta, feats, coords, init, idx = _problem(h=h, w=w)
    sc = FO.Scalars(0.01, 1, 1 if phase2 else 0, phase2, 1e-5, 1024.0)
    res = FO.step(init, feats, coords, idx[0], h, w, meta, sc)
    g32, out = _autograd(init, feats, coords, idx[0], h, w, meta, phase2, 1024.0)
    for k in ("loss", "patch_l2_loss", "cosine_similarity_loss") + (("residual_loss", "residual_sparsity_loss") if phase2 else ()):
        assert abs(res.losses[k] - out[k].item()) <= 1e-5 * abs(res.losses[k]), k
    names = [k for k in OF.PARAM_ORDER if res.trained[k]]
    assert set(names) == set(res.grad) and set(names) <= set(g32)
    for k in names:
        g, E, A = res.grad[k], res.env[k], res.allow[k]
        assert torch.all(g.abs() <= E * (1 + 1e-12) + A), f"{k}: the envelope does not bound the gradient"
        err = (g32[k].double() - g).abs()
        bound = res.c[k] * FO.U * E + A
        worst = float((err / (FO.U * E).clamp_min(1e-300)).max())
        print(f"{k:14s} c {res.c[k]:7.1f}  worst |g32 - g64| / (u E) {worst:8.2f}")
        assert torch.all(err <= bound), f"{k}: fp32 autograd outside c u E + A (worst ratio {worst:.1f}, c {res.c[k]:.1f})"
        assert (g.abs() > 0).any(), k


def test_oracle_keeps_the_neighbour_share_of_g():
    """On a 37 x 37 map grid_sample leaks ~1e-6 of 9 nodes per axis into a neighbouring cell: with 256 rows most cells are
    not any row's own cell, and those next to a leaking node still get their (tiny) share of the gradient, as in autograd."""
    h = w = 37
    meta, feats, coords, init, idx = _problem(C=32, h=h, w=w, V=1, bsz=256, L=4, T=1)
    sc = FO.Scalars(0.01, 1, 0, False, 1e-5, 1024.0)
    res = FO.step(init, feats, coords, idx[0], h, w, meta, sc)
    g32, _ = _autograd(init, feats, coords, idx[0], h, w, meta, False, 1024.0)
    own = torch.zeros(h * w, dtype=torch.bool)
    own[torch.as_tensor(idx[0]) % (h * w)] = True
    gG = res.grad["G"].reshape(-1, h * w)
    leak_only = (~own) & (gG.abs().sum(0) > 0)
    assert int(leak_only.sum()) >= 5
    share = gG[:, leak_only].abs().max() / gG[:, own].abs().max()
    assert 1e-8 < float(share) < 1e-5
    # the envelope of those cells is their own (tiny) size: autograd's fp32 share agrees to c u E there too
    err = (g32["G"].double().reshape(-1, h * w) - gG)[:, leak_only].abs()
    E = res.env["G"].reshape(-1, h * w)[:, leak_only]
    assert float(E.max()) < 1e-5 * float(res.env["G"].max())
    assert torch.all(err <= res.c["G"] * FO.U * E)


def _torch_adam_fp64(init, feats, coords, idx, h, w, meta, grads_of):
    """torch.optim.Adam in fp64, driven like OF.fit: lr set per step, G's requires_grad dropped at the freeze (grad None
    -> skipped), the residual MLP without a gradient until then.  grads_of(step, params) gives the fp64 gradients."""
    T = idx.shape[0]
    p = {k: init[k].clone().double().requires_grad_(True) for k in OF.PARAM_ORDER}
    opt = torch.optim.Adam([p[k] for k in OF.PARAM_ORDER], lr=HYPER["lr"], eps=1e-15,
                           weight_decay=HYPER["weight_decay"], betas=(0.9, 0.99))
    for s in range(T):
        sc = FO.scalars_at(s, num_iters=T, **HYPER)
        if sc.phase2:
            p["G"].requires_grad = False
        for grp in opt.param_groups:
            grp["lr"] = sc.lr
        opt.zero_grad()
        for k, g in grads_of(s, sc, {k: v.detach() for k, v in p.items()}).items():
            p[k].grad = g.clone()
        opt.step()
    return {k: v.detach() for k, v in p.items()}


def test_adam_restatement_reproduces_torch_adam_across_the_freeze():
    h, w = 6, 9
    meta, feats, coords, init, idx = _problem(h=h, w=w, T=6)
    T = idx.shape[0]
    cache = {}

    def grads_of(s, sc, p):
        if s not in cache:
            cache[s] = FO.step({k: v.float() for k, v in p.items()}, feats, coords, idx[s], h, w, meta, sc).grad
        return cache[s]

    # the restatement: p, m, v per tensor, counters from Scalars, G skipped in phase 2, residual only in phase 2
    p = {k: init[k].clone().double() for k in OF.PARAM_ORDER}
    m = {k: torch.zeros_like(v) for k, v in p.items()}
    v = {k: torch.zeros_like(x) for k, x in p.items()}
    freeze_step = int(HYPER["freeze_after"] * T)
    for s in range(T):
        sc = FO.scalars_at(s, num_iters=T, **HYPER)
        assert sc.phase2 == (s > freeze_step) and sc.tr == (s - freeze_step if sc.phase2 else 0)
        g = grads_of(s, sc, p)
        for k in OF.PARAM_ORDER:
            if not sc.phase2 and k in FO.RESIDUAL or sc.phase2 and k == "G":
                assert k not in g
                continue
            ss, ibc = sc.adam(k in FO.RESIDUAL)
            p[k], m[k], v[k] = FO.adam(p[k], m[k], v[k], g[k], ss, ibc, sc.wd)
    ref = _torch_adam_fp64(init, feats, coords, idx, h, w, meta, grads_of)
    for k in OF.PARAM_ORDER:
        d_ref, d_got = ref[k] - init[k].double(), p[k] - init[k].double()
        # the restatement rounds the per-step scalars to float like the engine's host code: 2^-24 relative per step
        # (each step moves an element by at most ~lr, so the rounding is bounded by that too)
        assert torch.allclose(d_got, d_ref, rtol=4 * 2.0 ** -24 * T, atol=4 * 2.0 ** -24 * T * HYPER["lr"]), \
            f"{k}: max update difference {(d_got - d_ref).abs().max().item()}"
        if k == "G":  # frozen after step freeze_step: only the phase-1 steps moved it
            assert (d_ref.abs() > 0).any()
    # and against OF.fit's own fp32 run (its own fp32 gradients): the same trajectory up to fp32 rounding
    ora = OF.fit(feats.reshape(-1, h, w, feats.shape[-1]), coords.reshape(-1, h, w, 2), h, w, meta, init, idx,
                 log_every=1, **HYPER)
    for k in OF.PARAM_ORDER:
        d32, d64 = ora["params"][k].double() - init[k].double(), p[k] - init[k].double()
        cos = torch.nn.functional.cosine_similarity(d32.flatten(), d64.flatten(), dim=0).item()
        # Adam's first steps move by ~lr * sign(g): an element whose gradient is within fp32 rounding of 0 may move the
        # other way, so the comparison is on the direction plus an element count, not elementwise
        close = ((d32 - d64).abs() <= 1e-6 * init[k].double().abs() + 1e-4 * HYPER["lr"]).double().mean().item()
        assert cos > 0.9999 and close > 0.99, f"{k}: cosine {cos}, fraction within rounding {close}"
