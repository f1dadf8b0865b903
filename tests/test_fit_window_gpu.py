"""Windowed table sweep (DVT_FIT_SWEEP_STEPS): the pipelined schedule that sweeps the hash table once per window of k
steps must give, bit for bit, what the sequential schedule (one sweep per step, in line) gives: the same table with its
Adam moments, the same small parameters and the same query output.  The logged losses are sums of float atomics (their
order is not fixed), so they are compared to rounding.  Fit lengths and phase boundaries are chosen so that neither is
a multiple of k, and graphs of 7 and 20 steps end inside windows, so every flush of a partial window is exercised."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SMALL = ("mlp.0.weight", "mlp.0.bias", "mlp.2.weight", "mlp.2.bias", "G", "res.0.weight", "res.0.bias", "res.2.weight",
         "res.2.bias", "res.4.weight", "res.4.bias")
HYPER = dict(lr=0.01, min_lr=0.001, freeze_after=0.5, weight_decay=1e-5, loss_scale=1024.0)


def _problem(C, h, w, V, bsz, n_levels, num_iters, seed):
    import dvt.models as DVT
    from oracle import fit as OF
    from oracle import hashgrid as HG
    feats, coords = OF.synthetic_bank(V, h, w, C, seed=seed)
    init = OF.init_params(C, h, w, HG.grid_meta(n_levels), seed=seed)
    idx = np.random.RandomState(seed).randint(0, V * h * w, (num_iters, bsz))
    field = DVT.NeuralFeatureField(feat_dim=C, n_levels=n_levels)
    return dict(C=C, h=h, w=w, bsz=bsz, meta=field.meta, feats=feats, coords=coords, init=init, idx=idx,
                warmup_iters=num_iters // 10)


def _fit(pb, monkeypatch, env, graph_steps, bank=None, coords=None, eng=None):
    """One fit under the DVT_FIT_* settings `env`; returns (engine, results)."""
    from dvt.fit import FitEngine
    for k in ("DVT_FIT_PIPELINE", "DVT_FIT_SWEEP_CTAS", "DVT_FIT_SWEEP_STEPS"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)                                 # read by dvt_fit_create
    C = pb["C"]
    if eng is None:
        eng = FitEngine(C, pb["h"], pb["w"], pb["bsz"], pb["meta"])
    for k, v in pb["init"].items():
        eng.set_param(k, v)
    bank = pb["feats"].reshape(-1, C).cuda().contiguous() if bank is None else bank
    coords = pb["coords"].reshape(-1, 2).cuda().contiguous() if coords is None else coords
    eng.begin(bank, coords, pb["idx"], warmup_iters=pb["warmup_iters"], **HYPER)
    eng.run(graph_steps=graph_steps)
    return eng, _results(eng, pb)


def _results(eng, pb):
    from dvt import _lib
    init = pb["init"]
    out = {"losses": eng.losses().copy(), "query": eng.query(pb["coords"][-1:].cuda()).cpu()}
    for k in ("table", "table.m", "table.v"):
        out[k] = eng.get_param(k, init["table"]).cpu()
    for k in SMALL:
        out[k] = eng.get_param(k, init[k]).cpu()
    torch.cuda.synchronize()
    assert _lib.device_error() == 0
    return out


def _assert_same(got, ref, what):
    assert np.allclose(got["losses"], ref["losses"], rtol=1e-5, atol=1e-7), f"{what}: losses differ"
    for k, v in ref.items():
        if k != "losses":
            assert torch.equal(got[k].view(torch.int32), v.view(torch.int32)), \
                f"{what}: {k} differs (max diff {(got[k] - v).abs().max().item()})"


_REF = {}


def _sequential(pb, key, monkeypatch):
    if key not in _REF:
        _REF[key] = _fit(pb, monkeypatch, {"DVT_FIT_PIPELINE": "0"}, 0)[1]
    return _REF[key]


@pytest.mark.parametrize("graph_steps", [0, 7, 20])
@pytest.mark.parametrize("k", [1, 2, 3, 4, 5, 8])
def test_windowed_sweep_matches_sequential(k, graph_steps, monkeypatch):
    # 16 levels (incl. hashed ones), 43 steps: phase 1 is steps 0..21 (22 steps), phase 2 has 21
    pb = _problem(C=64, h=6, w=6, V=4, bsz=128, n_levels=16, num_iters=43, seed=2)
    ref = _sequential(pb, "small", monkeypatch)
    _, got = _fit(pb, monkeypatch, {"DVT_FIT_SWEEP_STEPS": str(k), "DVT_FIT_SWEEP_CTAS": "6,3"}, graph_steps)
    _assert_same(got, ref, f"k={k} graph_steps={graph_steps}")


def test_windowed_sweep_per_phase_windows_and_full_grid(monkeypatch):
    """Different windows per phase, the many-CTA sweep geometry in phase 1 and the sequential schedule in phase 2."""
    pb = _problem(C=64, h=6, w=6, V=4, bsz=128, n_levels=16, num_iters=43, seed=2)
    ref = _sequential(pb, "small", monkeypatch)
    for env in ({"DVT_FIT_SWEEP_STEPS": "3,5", "DVT_FIT_SWEEP_CTAS": "0,4"},
                {"DVT_FIT_SWEEP_STEPS": "4,2", "DVT_FIT_SWEEP_CTAS": "5,-1"}):
        _, got = _fit(pb, monkeypatch, env, 7)
        _assert_same(got, ref, str(env))


def test_windowed_sweep_engine_reuse_with_another_bank(monkeypatch):
    """k = 4: a second fit on the same engine, with the bank in another buffer and the state buffers left by the first
    fit, equals a fit on a fresh engine."""
    pb = _problem(C=128, h=8, w=8, V=6, bsz=256, n_levels=6, num_iters=61, seed=0)
    C = pb["C"]
    env = {"DVT_FIT_SWEEP_STEPS": "4"}
    bank_a = (pb["feats"].reshape(-1, C) * -0.5 + 0.3).cuda().contiguous()
    coords_a = pb["coords"].reshape(-1, 2).flip(0).cuda().contiguous()
    eng, _ = _fit(pb, monkeypatch, env, 7, bank=bank_a, coords=coords_a)
    _, used = _fit(pb, monkeypatch, env, 7, eng=eng)
    _, fresh = _fit(pb, monkeypatch, env, 7)
    _assert_same(used, fresh, "reused engine")
    _assert_same(fresh, _fit(pb, monkeypatch, {"DVT_FIT_PIPELINE": "0"}, 7)[1], "k=4 vs sequential")


def test_sweep_once_applies_one_step(monkeypatch):
    """The measurement hook sweeps exactly one Adam step whatever the window: from zero moments and no gradient, weight
    decay 0.37 and lr 0.01 (no warm-up) move every parameter by lr / (1 - b1) * 0.1 * sign(p) = 0.01 sign(p)."""
    import dvt.models as DVT
    from dvt._lib import DvtError
    from dvt.fit import FitEngine
    C, h, w, bsz, L, T = 64, 6, 6, 128, 10, 8
    field = DVT.NeuralFeatureField(feat_dim=C, n_levels=L)
    g = torch.Generator(device="cuda").manual_seed(0)
    bank = torch.randn(4 * h * w, C, device="cuda", generator=g)
    co = torch.rand(4 * h * w, 2, device="cuda", generator=g)
    idx = np.random.RandomState(0).randint(0, 4 * h * w, (T, bsz))
    hyper = dict(lr=0.01, min_lr=0.001, warmup_iters=0, freeze_after=0.5, weight_decay=0.37, loss_scale=1024.0)
    outs = []
    for k, ctas in (("1", 7), ("4", 7), ("8", 0)):
        monkeypatch.setenv("DVT_FIT_SWEEP_STEPS", k)
        eng = FitEngine(C, h, w, bsz, field.meta)
        eng.init_params(5)
        eng.begin(bank, co, idx, **hyper)
        eng.sweep_once(ctas)
        start = eng.get_param("table", field.neural_field.params).cpu()
        outs.append(eng.get_param("table.next", field.neural_field.params).cpu())
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[1], outs[2])
    # (approximate sqrt / division inside adam1(); a second step would move every parameter by another 0.01)
    assert (outs[0] - (start - 0.01 * start.sign())).abs().max().item() < 1e-4
    with pytest.raises(DvtError):
        eng.sweep_once(-7)


def test_windowed_sweep_full_size(monkeypatch):
    """Headline size (C 768, 16 levels, 2048 pixels per step), 130 steps with the default window and 20-step graphs:
    the phase boundary (after step 65) falls inside a graph-sized block and a window."""
    pb = _problem(C=768, h=37, w=37, V=4, bsz=2048, n_levels=16, num_iters=130, seed=11)
    ref = _fit(pb, monkeypatch, {"DVT_FIT_PIPELINE": "0"}, 20)[1]
    _, got = _fit(pb, monkeypatch, {}, 20)
    _assert_same(got, ref, "default window, full size")
