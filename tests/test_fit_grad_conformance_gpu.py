"""Conformance of every gradient and Adam step of the stage-1 fit against fp64 (tests/fit_oracle_fp64.py), per step.

All steps are teacher-forced: the engine runs one plain step at a time (`run(1, graph_steps=0)`; graphs and sweep windows
are bit-identical to this, tests/test_fit_window_gpu.py), and step t is compared with the oracle evaluated at the engine's
own state S_t (p, m, v of all twelve tensors, read back with `get_param("<name>[.m|.v]")`).  Errors cannot compound, and a
failure names the step and the tensor.

The gradients are observed through Adam's first moment: the engine computes m_{t+1} = m_t + 0.1 (g' - m_t) with
g' = g + wd p_t in fp32, so g' = m_t + (m_{t+1} - m_t) / 0.1 up to the rounding of that one update (5 ulp(m_{t+1}) +
1.5 ulp(|g'| + |m_t|)).  At step 0 (lr 0 under warm-up) and at the residual MLP's first step, m_t = 0 and the read-back is
g' to one rounding.  Each gradient element must satisfy |g' - g'_64| <= c u E' + A (+ that read-back rounding), with
E' = E + wd |p_t| the envelope of g' and c, A as the oracle's docstring states them.  The decay-only table entries and the
neighbour share of G therefore get a tolerance proportional to their own size.

Schedule: 8 steps, warm-up 2, freeze_after 0.25: step 0 at lr 0, G frozen and the residual MLP trained from step 3.
Per step: the five logged losses within their error bounds (fp32 sums of up to 3 M terms, and pred's error: 2e-5 to
1e-3 relative, the most for the sparsity term at
C >= 1024, or with the SIMT GEMMs); every gradient within the envelope; m, v against the oracle's g' and p
against the engine's own m, v (ulp(p) + 2^-20 |step|: sqrt.approx and __fdividef); G bit-unchanged in phase 2; the
residual MLP bit-unchanged with m = v = 0 in phase 1; every p bit-unchanged at step 0.  After the last step `query()` and
`residual()` on the full-image view against fp64 at the engine's final parameters.

Each configuration prints the worst |g - g64| / (u E) per tensor (and its rms over the tensor, which must stay below
c / lambda: the error model in mean square), the number of elements that needed the ambiguity
allowance and its wall time."""
import time

import numpy as np
import pytest
import torch

import fit_oracle_fp64 as FO
from oracle import fit as OF
from oracle import hashgrid as HG

pytestmark = pytest.mark.gpu

T = 8
SCHED = dict(lr=0.01, min_lr=0.001, warmup_iters=2, freeze_after=0.25, weight_decay=1e-5, loss_scale=1024.0)
TENTH = float(np.float32(0.1))       # the engine's (1 - beta1) as a float
A_DOMINATED_MAX = 0.01               # at most 1 % of a tensor's elements may pass only through the allowance A


def _L():
    from dvt import _lib
    return _lib


def _state(eng, like):
    out = {}
    for k in OF.PARAM_ORDER:
        for suf in ("", ".m", ".v"):
            out[k + suf] = eng.get_param(k + suf, like[k]).cpu().double()
    return out


def _fail(what, bad, err, bound):
    i = int(torch.argmax((err - bound) * bad))
    return f"{what}: {int(bad.sum())} elements out of bound, worst at flat index {i}: |err| {err.flatten()[i]:.3e} > {bound.flatten()[i]:.3e}"


def _check_trained(tag, k, S, S1, ref, sc, report):
    p0, m0, v0, p1, m1, v1 = (X[k + s] for X in (S, S1) for s in ("", ".m", ".v"))
    wd = sc.wd
    g_ref = ref.grad[k] + wd * p0                                   # g' of the oracle
    E = ref.env[k] + wd * p0.abs()
    A = ref.allow[k]
    c = ref.c[k]
    g_eng = m0 + (m1 - m0) / TENTH                                  # g' of the engine
    rec = 5 * FO.ulp(m1) + 1.5 * FO.ulp(g_ref.abs() + m0.abs())
    err = (g_eng - g_ref).abs()
    bound = c * FO.U * E + A + rec
    bad = err > bound
    assert not bad.any(), _fail(f"{tag} gradient of {k} (c {c:.0f})", bad, err, bound)
    plain = (A == 0) & (E > 0)
    q = ((err - rec).clamp_min(0) / (FO.U * E).clamp_min(1e-300))[plain]
    ratio = float(q.max()) if q.numel() else 0.0
    # The same model in mean square (lambda = 1): over a whole tensor the rms of |g - g64| / (u E) stays below c / lambda.
    # This is what sees an error that is small per element but present in every element, e.g. a GEMM operand that lost
    # its lo plane (2^-12 relative per product, far below the per-element bound at K = 2048, but in every product).
    rms = float(q.square().mean().sqrt()) if q.numel() else 0.0
    assert rms <= c / FO.LAMBDA, f"{tag} {k}: rms of |g - g64| / (u E) is {rms:.1f} > c / lambda = {c / FO.LAMBDA:.1f}"
    dom = float((err > c * FO.U * E + rec).double().mean())      # elements that needed the allowance
    assert dom <= A_DOMINATED_MAX, f"{tag} {k}: {dom:.2%} of the elements pass only through the ambiguity allowance"
    r = report.setdefault(k, [0.0, c, 0.0])
    r[0], r[1], r[2] = max(r[0], ratio), max(r[1], c), max(r[2], rms)
    # second moment against the oracle's g' (its error bounded by the gradient bound)
    tol_g = c * FO.U * E + A
    v_ref = 0.99 * v0 + 0.01 * g_ref * g_ref
    err_v = (v1 - v_ref).abs()
    bound_v = 0.01 * (2 * g_ref.abs() * tol_g + tol_g * tol_g) + 4 * FO.ulp(v1) + 4 * FO.ulp(v_ref)
    bad = err_v > bound_v
    assert not bad.any(), _fail(f"{tag} second moment of {k}", bad, err_v, bound_v)
    # parameter update from the engine's own m, v
    ss, ibc = sc.adam(k in FO.RESIDUAL)
    stp = ss * m1 / (v1.sqrt() * ibc + 1e-15)
    err_p = (p1 - (p0 - stp)).abs()
    bound_p = torch.maximum(FO.ulp(p0), FO.ulp(p1)) + 2.0 ** -20 * stp.abs()
    bad = err_p > bound_p
    assert not bad.any(), _fail(f"{tag} update of {k}", bad, err_p, bound_p)
    if sc.lr == 0:
        assert torch.equal(p1, p0), f"{tag} {k} moved at lr 0"


def _check_frozen(tag, k, S, S1, zero_moments):
    for s in ("", ".m", ".v"):
        assert torch.equal(S1[k + s], S[k + s]), f"{tag} {k}{s} changed while {k} is not trained"
        if zero_moments and s:
            assert not S1[k + s].any(), f"{tag} {k}{s} is not zero before the residual MLP's first step"


def _run(C, h, w, *, bsz=2048, L=16, simt=False, exact=True, seed=17, V=2):
    from dvt.fit import FitEngine
    from dvt.models.hashgrid_meta import make_meta
    t_start = time.time()
    meta, ometa = make_meta(L), HG.grid_meta(L)
    feats, coords = OF.synthetic_bank(V, h, w, C, seed=seed)
    feats, coords = feats.reshape(-1, C), coords.reshape(-1, 2)
    init = OF.init_params(C, h, w, ometa, seed=seed)
    idx = np.random.RandomState(seed).randint(0, V * h * w, (T, bsz))
    eng = FitEngine(C, h, w, bsz, meta)
    for k, v in init.items():
        eng.set_param(k, v)
    L_ = _L()
    L_.check(L_.lib().dvt_set_debug_impl(1 if simt else -1))
    try:
        eng.begin(feats.cuda().contiguous(), coords.cuda().contiguous(), idx, **SCHED)
        S = _state(eng, init)
        report, n_amb = {}, 0
        for t in range(T):
            sc = FO.scalars_at(t, num_iters=T, **SCHED)
            ref = FO.step({k: S[k].float() for k in OF.PARAM_ORDER}, feats, coords, idx[t], h, w, ometa, sc,
                          exact_grid=exact, simt=simt)
            eng.run(1, graph_steps=0)
            S1 = _state(eng, init)
            assert L_.device_error() == 0
            tag = f"step {t}"
            got = eng.losses()[t]
            for j, name in enumerate(("loss", "patch_l2_loss", "cosine_similarity_loss", "residual_loss",
                                      "residual_sparsity_loss")):
                want = ref.losses[name]
                tol = ref.loss_tol[name]
                assert tol <= 2e-3 * abs(want) + 1e-9, f"{tag} {name}: the error bound {tol} is no test"
                assert abs(float(got[j]) - want) <= tol, f"{tag} {name}: {got[j]} vs fp64 {want} (bound {tol:.2e})"
            for k in OF.PARAM_ORDER:
                if ref.trained[k]:
                    _check_trained(tag, k, S, S1, ref, sc, report)
                else:
                    _check_frozen(tag, k, S, S1, zero_moments=k in FO.RESIDUAL)
            n_amb += ref.n_ambiguous
            S = S1
        # final outputs at the engine's parameters, on the full-image view (the bank's last view)
        p = {k: S[k].float() for k in OF.PARAM_ORDER}
        full_c = coords.reshape(V, h * w, 2)[-1]
        full_r = feats.reshape(V, h * w, C)[-1]
        for what, got, (y, yE, c) in (("query", eng.query(full_c.cuda()), FO.query_ref(p, full_c, ometa, simt)),
                                      ("residual", eng.residual(full_r.cuda()), FO.residual_ref(p, full_r, simt))):
            err = (got.cpu().double() - y).abs()
            bound = c * FO.U * yE
            bad = err > bound
            assert not bad.any(), _fail(f"final {what} (c {c:.0f})", bad, err, bound)
            report[what] = [float((err / (FO.U * yE).clamp_min(1e-300)).max()), c, float("nan")]
        assert L_.device_error() == 0
    finally:
        L_.check(L_.lib().dvt_set_debug_impl(-1))
    worst = ", ".join(f"{k} {r:.2f}/{q:.2f}/{c:.0f}" for k, (r, c, q) in report.items())
    print(f"\n[fit conformance C {C} map {h}x{w} bsz {bsz} L {L}{' simt' if simt else ''}{'' if exact else ' plain-grid'}] "
          f"worst |g - g64| / (u E), its rms, c: {worst}; ambiguous elements {n_amb}; {time.time() - t_start:.1f} s")
    return report


# The big widths run the loss kernel's 8- and 12-vector instances, the G scatter with more than 6 float4 per lane and the
# 128-wide weight-gradient tiles at N = C / 2 + 1 and C + 1; they carry the `wide` keyword so that the file splits into
# groups of tests/run_gpu_groups.sh.
CONFIGS = {
    "C384": dict(C=384, h=37, w=37),
    "C768": dict(C=768, h=37, w=37),
    "wide_C1024": dict(C=1024, h=37, w=37),
    "wide_C1280": dict(C=1280, h=37, w=37),
    "wide_C1536": dict(C=1536, h=37, w=37),
    "C1024_23x31": dict(C=1024, h=23, w=31),         # non-square map: axis tables, cell / gw, G's transpose
    "C768_bsz1000": dict(C=768, h=37, w=37, bsz=1000),  # M / K tails of the transposed planes
    "C96_6x9": dict(C=96, h=6, w=9),                 # partial float4 lanes, tiny C / 4 GEMMs
    "C160_6x9": dict(C=160, h=6, w=9),
    "C32_6x9": dict(C=32, h=6, w=9),                 # the smallest width fit_create accepts
    "C768_L10": dict(C=768, h=37, w=37, L=10),       # K = 80 for mlp.0, the class default
}


@pytest.mark.parametrize("name", list(CONFIGS))
def test_fit_step_conformance(name):
    _run(**CONFIGS[name])


def test_fit_step_conformance_plain_grid(monkeypatch):
    """DVT_FIT_EXACT_GRID=0: the plain cell indexing of the loss and the G scatter (weight 1 on the node's own cell)."""
    monkeypatch.setenv("DVT_FIT_EXACT_GRID", "0")
    _run(768, 37, 37, exact=False)


def test_fit_step_conformance_simt():
    """The SIMT debug GEMMs (dvt_set_debug_impl(1)) honour the same contract, with their own accumulation depth."""
    _run(1024, 37, 37, simt=True)


@pytest.mark.parametrize("sms", ["1", "13", "96", "132"])
def test_fit_step_conformance_wgrad_partition(sms, monkeypatch):
    """Every split-K partition of the weight-gradient GEMMs (DVT_FIT_WGRAD_SMS) is fp32-accurate, not just the default."""
    monkeypatch.setenv("DVT_FIT_WGRAD_SMS", sms)
    _run(1024, 37, 37)
