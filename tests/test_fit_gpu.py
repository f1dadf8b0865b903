"""HP-2 parity on the GPU: hash-grid indexing (bit-exact) and encoding against oracle/hashgrid.py, MN-major GEMM
variants against torch, and the fused per-image fit against the golden fixtures that
tests/golden/make_fit_golden.py produced with the REFERENCE's SingleImageDenoiser + torch Adam loop.

Tolerances: indices / interpolation weights bit-exact; denoised features cosine >= 0.999 per patch
(BASELINE.json north_star); loss trajectory within 2 % (3xTF32 tensor-core GEMMs and another summation order vs fp32 CPU)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _L():
    from dvt import _lib
    return _lib


class _impl:
    def __init__(self, impl):
        self.impl = impl

    def __enter__(self):
        L = _L()
        L.check(L.lib().dvt_set_debug_impl(self.impl))

    def __exit__(self, *a):
        L = _L()
        L.check(L.lib().dvt_set_debug_impl(-1))


def _coords(n, seed):
    g = torch.Generator().manual_seed(seed)
    c = torch.rand(n, 2, generator=g)
    edge = torch.tensor([[0.0, 0.0], [1.0, 1.0], [0.0, 1.0], [1.0, 0.0], [0.5, 0.5], [1.0 / 3, 2.0 / 3],
                         [0.999999, 0.000001], [15.5 / 16, 0.25]])
    c[:edge.shape[0]] = edge
    return c


@pytest.mark.parametrize("n_levels", [6, 10, 16])
def test_hashgrid_indexing_bit_exact(n_levels):
    from dvt._lib import check, cur_stream, lib, ptr
    from dvt.models.hashgrid_meta import make_meta
    from oracle import hashgrid as HG
    meta, ometa = make_meta(n_levels), HG.grid_meta(n_levels)
    n = 4096
    c = _coords(n, n_levels)
    cd = c.cuda()
    idx = torch.zeros(n, n_levels, 4, dtype=torch.int32, device="cuda")
    w = torch.zeros(n, n_levels, 4, dtype=torch.float32, device="cuda")
    check(lib().dvt_hashgrid_corners(*meta.c_args(), ptr(cd), n, ptr(idx), ptr(w), cur_stream()))
    torch.cuda.synchronize()
    for l in range(n_levels):
        oi, ow = HG.corner_indices_weights(c, ometa, l)
        got_i = idx[:, l].cpu().to(torch.int64) & 0xFFFFFFFF
        assert torch.equal(got_i, oi + int(ometa.offset[l])), f"level {l}: corner indices differ"
        assert torch.equal(w[:, l].cpu(), ow), f"level {l}: interpolation weights differ"


@pytest.mark.parametrize("n_levels", [6, 16])
def test_hashgrid_fwd_bwd(n_levels):
    import dvt.models as DVT
    from oracle import hashgrid as HG
    ometa = HG.grid_meta(n_levels)
    field = DVT.NeuralFeatureField(feat_dim=64, n_levels=n_levels).cuda()
    table = field.neural_field.params.detach().cpu() * 1e3  # O(0.1) values
    with torch.no_grad():
        field.neural_field.params.copy_(table.cuda())
    c = _coords(2048, 7)
    ref_t = table.clone().requires_grad_(True)
    ref = HG.encode(ref_t, c, ometa)
    got = field.neural_field(c.cuda())
    assert torch.allclose(got.cpu(), ref.detach(), rtol=1e-5, atol=1e-6)
    dout = torch.randn(ref.shape, generator=torch.Generator().manual_seed(1))
    ref.backward(dout)
    got.backward(dout.cuda())
    g = field.neural_field.params.grad.cpu()
    assert torch.allclose(g, ref_t.grad, rtol=1e-4, atol=1e-5), (g - ref_t.grad).abs().max()


@pytest.mark.parametrize("impl", [1, 0], ids=["simt", "tcgen05"])
def test_gemm_mn_major(impl):
    from dvt import ops
    g = torch.Generator(device="cuda").manual_seed(3)
    n, C, H1 = 2048, 768, 384
    dy = torch.randn(n, C, device="cuda", generator=g).bfloat16()
    x = torch.randn(n, H1 + 8, device="cuda", generator=g).bfloat16()
    x[:, H1] = 1.0
    w = (torch.randn(C, H1, device="cuda", generator=g) / 20).bfloat16()
    with _impl(impl):
        # dgrad: dX[n, H1] = dY[n, C] . W[C, H1]  (B = W read as MN-major)
        dx = ops.gemm_bf16_ex(dy, w, n, H1, C, a_mn=False, b_mn=True)
        # wgrad + bias grad: dW[C, H1] | db[C] = dY^T . [X | 1]
        dw, db = ops.gemm_bf16_ex(dy, x, C, H1 + 1, n, a_mn=True, b_mn=True, splits=8, last_col=True)
        # ragged: K = 200 rows, N = 129
        dy2, x2 = dy[:200, :256].contiguous(), x[:200, :136].contiguous()
        dw2, db2 = ops.gemm_bf16_ex(dy2, x2, 256, 129, 200, a_mn=True, b_mn=True, splits=1, last_col=True)
    torch.cuda.synchronize()
    assert (dx - dy.float() @ w.float()).abs().max().item() < 2e-2
    ref = dy.float().t() @ x[:, :H1 + 1].float()
    assert (dw - ref[:, :H1]).abs().max().item() < 0.15
    assert (db - ref[:, H1]).abs().max().item() < 0.15
    ref2 = dy2.float().t() @ x2[:, :129].float()
    assert (dw2 - ref2[:, :128]).abs().max().item() < 5e-2
    assert (db2 - ref2[:, 128]).abs().max().item() < 5e-2
    assert _L().device_error() == 0


@pytest.mark.parametrize("impl", [1, 0], ids=["simt", "tcgen05"])
def test_gemm_f32x3_is_fp32_accurate(impl):
    """3xTF32 on the tensor cores must match an fp64 reference to fp32 accuracy (plain TF32 would be ~1e-3)."""
    from dvt import ops
    g = torch.Generator(device="cuda").manual_seed(9)
    n, C, H1 = 2048, 768, 384
    x = torch.randn(n, H1 + 8, device="cuda", generator=g)
    x[:, H1] = 1.0
    w = torch.randn(C, H1, device="cuda", generator=g) / 20
    dy = torch.randn(n, C, device="cuda", generator=g)
    with _impl(impl):
        y = ops.gemm_f32x3(x[:, :H1].contiguous(), w, n, C, H1)                               # forward  X W^T
        dx = ops.gemm_f32x3(dy, w, n, H1, C, a_mn=False, b_mn=True)                            # dgrad    dY W
        dw, db = ops.gemm_f32x3(dy, x, C, H1 + 1, n, a_mn=True, b_mn=True, splits=8, last_col=True)  # wgrad dY^T [X|1]
        dy2, x2 = dy[:200, :256].contiguous(), x[:200, :136].contiguous()
        dw2, db2 = ops.gemm_f32x3(dy2, x2, 256, 129, 200, a_mn=True, b_mn=True, splits=1, last_col=True)
    torch.cuda.synchronize()

    def rel(a, b):
        return ((a.double() - b).norm() / b.norm()).item()
    ref = dy.double().t() @ x[:, :H1 + 1].double()
    ref2 = dy2.double().t() @ x2[:, :129].double()
    errs = {"fwd(K,K)": rel(y, x[:, :H1].double() @ w.double().t()), "dgrad(K,MN)": rel(dx, dy.double() @ w.double()),
            "wgrad(MN,MN)": rel(dw, ref[:, :H1]), "bgrad": rel(db, ref[:, H1]), "wgrad ragged": rel(dw2, ref2[:, :128]),
            "bgrad ragged": rel(db2, ref2[:, 128])}
    bad = {k: v for k, v in errs.items() if not v < 1e-5}
    assert not bad, f"relative errors vs fp64: {errs}"
    assert _L().device_error() == 0


def _golden(name):
    z = np.load(os.path.join(GOLD, f"fit_{name}.npz"))
    parts = sorted(f for f in os.listdir(GOLD) if f.startswith(f"fit_{name}_part") and f.endswith(".npz"))
    if parts:  # the denoised map stored in row bands (files under 1 MB): join them
        bands = [z["denoised_feats"]] + [np.load(os.path.join(GOLD, f))["denoised_feats"] for f in parts]
        z = {**{k: z[k] for k in z.files}, "denoised_feats": np.concatenate(bands, axis=1)}
    cfg = {k: v for k, v in zip(z["cfg_keys"], z["cfg_vals"])}
    for k in ("C", "h", "w", "V", "bsz", "n_levels", "num_iters", "warmup_iters", "log_every", "seed"):
        cfg[k] = int(cfg[k])
    return cfg, z


def _setup(cfg):
    """Same seeded inputs / initial parameters as tests/golden/make_fit_golden.py."""
    import dvt.models as DVT
    from oracle import fit as OF
    from oracle import hashgrid as HG
    ometa = HG.grid_meta(cfg["n_levels"])
    feats, coords = OF.synthetic_bank(cfg["V"], cfg["h"], cfg["w"], cfg["C"], seed=cfg["seed"])
    init = OF.init_params(cfg["C"], cfg["h"], cfg["w"], ometa, seed=cfg["seed"])
    idx = np.random.RandomState(cfg["seed"]).randint(0, cfg["V"] * cfg["h"] * cfg["w"], (cfg["num_iters"], cfg["bsz"]))
    den = DVT.SingleImageDenoiser(cfg["h"], cfg["w"], cfg["C"], layer_index=11)
    field = DVT.NeuralFeatureField(feat_dim=cfg["C"], n_levels=cfg["n_levels"])
    with torch.no_grad():
        den.shared_artifacts.copy_(init["G"])
        for i in (0, 2, 4):
            den.residual_predictor[i].weight.copy_(init[f"res.{i}.weight"])
            den.residual_predictor[i].bias.copy_(init[f"res.{i}.bias"])
        field.neural_field.params.copy_(init["table"])
        for i in (0, 2):
            field.mlp[i].weight.copy_(init[f"mlp.{i}.weight"])
            field.mlp[i].bias.copy_(init[f"mlp.{i}.bias"])
    return feats, coords, init, idx, den.cuda(), field.cuda(), ometa


def _min_cos(a, b):
    return F.cosine_similarity(a.float().reshape(-1, a.shape[-1]), b.float().reshape(-1, b.shape[-1]), dim=-1).min().item()


@pytest.mark.parametrize("impl,graph_steps,pipeline", [(1, 0, 1), (0, 0, 1), (0, 7, 1), (0, 7, 0), (0, 0, 0)],
                         ids=["simt", "tcgen05", "tcgen05-graphs", "tcgen05-graphs-sequential", "tcgen05-sequential"])
@pytest.mark.parametrize("name", ["small_L6", "small_L6_ls1", "hashed_L16"])
def test_fit_matches_reference_golden(name, impl, graph_steps, pipeline, monkeypatch):
    """pipeline=1: default schedule (table sweeps run two steps behind the chain, Adam applied on the fly by the
    encode); pipeline=0: sequential schedule.  Both must reproduce the reference run."""
    from dvt.fit import FitEngine
    monkeypatch.setenv("DVT_FIT_PIPELINE", str(pipeline))   # read by dvt_fit_create
    monkeypatch.setenv("DVT_FIT_SWEEP_CTAS", "6,3")         # pipelined in both phases (the default is phase 1 only)
    cfg, z = _golden(name)
    feats, coords, init, idx, den, field, _ = _setup(cfg)
    assert int(idx.sum()) == int(z["idx_checksum"][0])  # same sampling stream as the reference run
    eng = FitEngine(cfg["C"], cfg["h"], cfg["w"], cfg["bsz"], field.meta)
    bank = feats.reshape(-1, cfg["C"]).cuda().contiguous()
    bcoords = coords.reshape(-1, 2).cuda().contiguous()
    with _impl(impl):
        eng.fit(den, field, bank, bcoords, idx, graph_steps=graph_steps, lr=cfg["lr"], min_lr=cfg["min_lr"],
                warmup_iters=cfg["warmup_iters"], freeze_after=cfg["freeze_after"], weight_decay=cfg["weight_decay"],
                loss_scale=cfg["loss_scale"])
        denoised = eng.query(coords[-1:].cuda())                       # [1, h, w, C]
        resid = eng.residual(feats[-1:].cuda())
    torch.cuda.synchronize()
    assert _L().device_error() == 0
    ref_feats = torch.from_numpy(z["denoised_feats"])
    mc = _min_cos(denoised.cpu(), ref_feats)
    assert mc > 0.999, f"denoised_feats min cosine {mc}"
    # loss trajectory at the steps the reference logged
    losses = eng.losses()
    logs = z["logs"]
    for row in logs:
        s = int(row[0])
        for j in range(5):
            ref_v, got_v = row[1 + j], losses[s, j]
            assert abs(got_v - ref_v) <= 0.02 * abs(ref_v) + 1e-3, f"step {s} loss[{j}] {got_v} vs {ref_v}"
    # "real denoised feature map" raw - G - residual (offline_denoiser.py:163-169)
    G = eng.get_param("G", den.shared_artifacts).permute(0, 2, 3, 1).cpu()
    got_clean = feats[-1:] - G - resid.cpu()
    assert _min_cos(got_clean, torch.from_numpy(z["denoised_features"])) > 0.999
    assert (G.permute(0, 3, 1, 2) - torch.from_numpy(z["G_final"])).abs().max().item() < 0.05
    # parameters flow back into the drop-in modules
    eng.store_modules(den, field)
    assert torch.isfinite(field.neural_field.params).all()
    tsum = float(field.neural_field.params.double().sum())
    assert abs(tsum - float(z["table_sum"][0])) <= 0.02 * float(z["table_sum"][1]) + 1e-3


def test_fit_is_bit_exact_run_to_run():
    """Two fits from the same inputs and initial parameters give bit-identical results.  The size makes every reduction of
    the step collide: 2048 samples per step on 16 hash-grid levels (coarse levels: many samples per entry), 2048 rows
    on 256 cells of G, split-K weight-gradient GEMMs.  Float atomics there would make the result depend on scheduling, and
    Adam turns that into visibly different fits."""
    from dvt.fit import FitEngine
    cfg = {"C": 384, "V": 8, "h": 16, "w": 16, "bsz": 2048, "n_levels": 16, "num_iters": 60, "seed": 5}
    outs = []
    for _ in range(2):
        feats, coords, init, idx, den, field, _ = _setup(cfg)
        eng = FitEngine(cfg["C"], cfg["h"], cfg["w"], cfg["bsz"], field.meta)
        eng.fit(den, field, feats.reshape(-1, cfg["C"]).cuda().contiguous(), coords.reshape(-1, 2).cuda().contiguous(), idx,
                graph_steps=20, lr=0.01, min_lr=0.001, warmup_iters=6, freeze_after=0.5, weight_decay=1e-5, loss_scale=1024.0)
        denoised = eng.query(coords[-1:].cuda()).cpu()
        G = eng.get_param("G", den.shared_artifacts).cpu()
        eng.store_modules(den, field)
        torch.cuda.synchronize()
        outs.append((denoised, G, field.neural_field.params.detach().cpu().clone(), field.mlp[0].weight.detach().cpu().clone()))
        del eng
    assert _L().device_error() == 0
    for k, (a, b) in enumerate(zip(*outs)):
        assert torch.equal(a, b), f"output {k} differs between two identical fits (max diff {(a - b).abs().max().item()})"


@pytest.mark.parametrize("impl", [1, 0], ids=["simt", "tcgen05"])
def test_fit_first_steps_update_direction(impl):
    """Three optimisation steps against the CPU oracle: every parameter group must move in the oracle's direction
    (Adam's first steps are ~ lr * sign(grad), so this checks gradients, schedules and the freeze logic)."""
    from dvt.fit import FitEngine
    from oracle import fit as OF
    cfg = dict(C=128, h=8, w=8, V=6, bsz=256, n_levels=6, num_iters=4, warmup_iters=2, lr=0.01, min_lr=0.001,
               weight_decay=1e-5, freeze_after=0.5, loss_scale=1024.0, seed=5)
    feats, coords, init, idx, den, field, ometa = _setup(cfg)
    ora = OF.fit(feats, coords, cfg["h"], cfg["w"], ometa, init, idx, lr=cfg["lr"], min_lr=cfg["min_lr"],
                 weight_decay=cfg["weight_decay"], warmup_iters=cfg["warmup_iters"], freeze_after=cfg["freeze_after"],
                 loss_scale=cfg["loss_scale"])
    eng = FitEngine(cfg["C"], cfg["h"], cfg["w"], cfg["bsz"], field.meta)
    with _impl(impl):
        eng.fit(den, field, feats.reshape(-1, cfg["C"]).cuda().contiguous(), coords.reshape(-1, 2).cuda().contiguous(),
                idx, graph_steps=0, lr=cfg["lr"], min_lr=cfg["min_lr"], warmup_iters=cfg["warmup_iters"],
                freeze_after=cfg["freeze_after"], weight_decay=cfg["weight_decay"], loss_scale=cfg["loss_scale"])
    torch.cuda.synchronize()
    names = {"G": init["G"], "table": init["table"], "mlp.0.weight": init["mlp.0.weight"],
             "mlp.2.weight": init["mlp.2.weight"], "mlp.2.bias": init["mlp.2.bias"], "res.4.weight": init["res.4.weight"],
             "res.0.weight": init["res.0.weight"], "res.2.bias": init["res.2.bias"]}
    for k, p0 in names.items():
        got = eng.get_param(k, p0).cpu() - p0
        ref = ora["params"][k] - p0
        moved = ref.abs() > 0
        assert moved.any(), k
        cos = F.cosine_similarity(got[moved].flatten(), ref[moved].flatten(), dim=0).item()
        assert cos > 0.9, f"{k}: update direction cosine {cos}"
        assert abs(got.abs().max().item() - ref.abs().max().item()) < 0.2 * ref.abs().max().item() + 1e-6, k
    assert _L().device_error() == 0


@pytest.mark.parametrize("sweep_ctas", ["0", "8,4", "4,-1", "-1,0"])
def test_fit_schedules_agree(sweep_ctas, monkeypatch):
    """The software-pipelined schedule is an exact re-ordering: after the same steps its table must equal the sequential
    schedule's within the tolerance below."""
    from dvt.fit import FitEngine
    cfg, z = _golden("hashed_L16")
    outs = []
    for pipeline in ("0", "1"):
        monkeypatch.setenv("DVT_FIT_PIPELINE", pipeline)
        monkeypatch.setenv("DVT_FIT_SWEEP_CTAS", sweep_ctas)
        feats, coords, init, idx, den, field, _ = _setup(cfg)
        eng = FitEngine(cfg["C"], cfg["h"], cfg["w"], cfg["bsz"], field.meta)
        eng.fit(den, field, feats.reshape(-1, cfg["C"]).cuda().contiguous(), coords.reshape(-1, 2).cuda().contiguous(), idx,
                graph_steps=5, lr=cfg["lr"], min_lr=cfg["min_lr"], warmup_iters=cfg["warmup_iters"],
                freeze_after=cfg["freeze_after"], weight_decay=cfg["weight_decay"], loss_scale=cfg["loss_scale"])
        torch.cuda.synchronize()
        outs.append((eng.get_param("table", init["table"]).cpu() - init["table"], eng.losses().copy()))
        assert _L().device_error() == 0
    (ta, la), (tb, lb) = outs
    cos = F.cosine_similarity(ta.flatten().double(), tb.flatten().double(), dim=0).item()
    assert cos > 0.9999, f"table update cosine between schedules {cos}"
    assert np.allclose(la, lb, rtol=1e-3, atol=1e-5)


def test_fit_engine_reuse_with_another_bank():
    """A second fit on the same engine with the bank in ANOTHER buffer (the stage-1 pipeline alternates two) must replay
    its captured CUDA graphs against the new bank: same result as a fresh engine."""
    from dvt.fit import FitEngine
    cfg, z = _golden("small_L6")
    feats, coords, init, idx, den, field, _ = _setup(cfg)
    hyper = dict(graph_steps=7, lr=cfg["lr"], min_lr=cfg["min_lr"], warmup_iters=cfg["warmup_iters"],
                 freeze_after=cfg["freeze_after"], weight_decay=cfg["weight_decay"], loss_scale=cfg["loss_scale"])
    bank_a = (feats.reshape(-1, cfg["C"]) * -0.5 + 0.3).cuda().contiguous()     # some other image
    bank_b = feats.reshape(-1, cfg["C"]).cuda().contiguous()
    coords_a = coords.reshape(-1, 2).flip(0).cuda().contiguous()
    coords_b = coords.reshape(-1, 2).cuda().contiguous()
    assert bank_a.data_ptr() != bank_b.data_ptr() and coords_a.data_ptr() != coords_b.data_ptr()
    used = FitEngine(cfg["C"], cfg["h"], cfg["w"], cfg["bsz"], field.meta)
    used.fit(den, field, bank_a, coords_a, idx, **hyper)
    used.fit(den, field, bank_b, coords_b, idx, **hyper)       # graphs captured by the first fit are replayed here
    fresh = FitEngine(cfg["C"], cfg["h"], cfg["w"], cfg["bsz"], field.meta)
    fresh.fit(den, field, bank_b, coords_b, idx, **hyper)
    torch.cuda.synchronize()
    assert _L().device_error() == 0
    qa, qb = used.query(coords[-1:].cuda()), fresh.query(coords[-1:].cuda())
    assert _min_cos(qa.cpu(), qb.cpu()) > 0.9999
    assert _min_cos(qa.cpu(), torch.from_numpy(z["denoised_feats"])) > 0.999
    assert np.allclose(used.losses(), fresh.losses(), rtol=1e-3, atol=1e-5)


# ---- headline problem size (BASELINE.json configs[2]: C 768, 37 x 37 noise map, 16 levels incl. the hashed one,
# ---- 2048 pixels per step); small synthetic bank so that the CPU oracle finishes in seconds ----------------------
_FULL = dict(C=768, h=37, w=37, V=4, bsz=2048, n_levels=16, lr=0.01, min_lr=0.001, weight_decay=1e-5, freeze_after=0.5,
             loss_scale=1024.0, seed=11)


def test_fit_full_size_first_steps_match_oracle():
    """Six optimisation steps at the headline size against the CPU oracle (three per phase): logged losses within 1e-3
    relative, every parameter group moves along the oracle's update."""
    from dvt.fit import FitEngine
    from oracle import fit as OF
    cfg = dict(_FULL, num_iters=6, warmup_iters=2)
    feats, coords, init, idx, den, field, ometa = _setup(cfg)
    ora = OF.fit(feats, coords, cfg["h"], cfg["w"], ometa, init, idx, lr=cfg["lr"], min_lr=cfg["min_lr"],
                 weight_decay=cfg["weight_decay"], warmup_iters=cfg["warmup_iters"], freeze_after=cfg["freeze_after"],
                 loss_scale=cfg["loss_scale"], log_every=1)
    eng = FitEngine(cfg["C"], cfg["h"], cfg["w"], cfg["bsz"], field.meta)
    eng.fit(den, field, feats.reshape(-1, cfg["C"]).cuda().contiguous(), coords.reshape(-1, 2).cuda().contiguous(), idx,
            graph_steps=2, lr=cfg["lr"], min_lr=cfg["min_lr"], warmup_iters=cfg["warmup_iters"],
            freeze_after=cfg["freeze_after"], weight_decay=cfg["weight_decay"], loss_scale=cfg["loss_scale"])
    torch.cuda.synchronize()
    assert _L().device_error() == 0
    losses = eng.losses()
    for row in ora["logs"]:
        s = int(row[0])
        for j in range(5):
            assert abs(losses[s, j] - row[1 + j]) <= 1e-3 * abs(row[1 + j]) + 1e-6, f"step {s} loss[{j}] {losses[s, j]} vs {row[1 + j]}"
    for k in ("table", "G", "mlp.0.weight", "mlp.2.weight", "res.0.weight", "res.4.weight"):
        got = eng.get_param(k, init[k]).cpu() - init[k]
        ref = ora["params"][k] - init[k]
        moved = ref.abs() > 0
        cos = F.cosine_similarity(got[moved].flatten().double(), ref[moved].flatten().double(), dim=0).item()
        assert cos > 0.99, f"{k}: update cosine {cos} at the headline size"


def test_fit_full_size_schedules_agree(monkeypatch):
    """Size-independent property at the headline size: the software-pipelined schedule (default) and the sequential one
    are the same computation -- 80 steps across the phase boundary give the same table and the same loss trajectory."""
    from dvt.fit import FitEngine
    cfg = dict(_FULL, num_iters=80, warmup_iters=8)
    outs = []
    for pipeline in ("0", "1"):
        monkeypatch.setenv("DVT_FIT_PIPELINE", pipeline)
        feats, coords, init, idx, den, field, _ = _setup(cfg)
        eng = FitEngine(cfg["C"], cfg["h"], cfg["w"], cfg["bsz"], field.meta)
        eng.fit(den, field, feats.reshape(-1, cfg["C"]).cuda().contiguous(), coords.reshape(-1, 2).cuda().contiguous(), idx,
                graph_steps=20, lr=cfg["lr"], min_lr=cfg["min_lr"], warmup_iters=cfg["warmup_iters"],
                freeze_after=cfg["freeze_after"], weight_decay=cfg["weight_decay"], loss_scale=cfg["loss_scale"])
        torch.cuda.synchronize()
        assert _L().device_error() == 0
        outs.append((eng.get_param("table", init["table"]).cpu() - init["table"], eng.losses().copy(),
                     eng.query(coords[-1:].cuda()).cpu()))
    (ta, la, qa), (tb, lb, qb) = outs
    cos = F.cosine_similarity(ta.flatten().double(), tb.flatten().double(), dim=0).item()
    assert cos > 0.9999, f"table update cosine between schedules {cos}"
    assert np.allclose(la, lb, rtol=2e-3, atol=1e-5)
    assert _min_cos(qa, qb) > 0.9999
    assert la[-1, 0] < la[8, 0], "the loss must fall over the run"


def test_fit_headline_2000_steps_matches_reference_golden():
    """THE full-length trajectory at the headline size (SURVEY.md 8(c)): C 768, 37 x 37, 16 levels (19.7 M-entry table with
    the hashed level), 2048 pixels per step, 2000 steps across the phase boundary, default schedule knobs (software-
    pipelined sweep, CUDA graphs of 20 steps), against the run of the REFERENCE's own SingleImageDenoiser + torch Adam
    loop stored by tests/golden/make_fit_golden_headline.py.

    Tolerances and where they come from.  2000 Adam steps on 21 M parameters amplify rounding noise: Adam normalises every
    gradient, so an element whose gradient is ~0 moves by +-lr on the sign of the noise.  Noise floors at exactly this
    configuration:
      * the reference against ITSELF with the 2048 rows of every step visited in another order (tools/oracle_noise_floor.py,
        CPU, mathematically the identical run): per-patch cosine min 0.99912 / mean 0.99988, logged losses within 2.9 %;
      * this engine against itself, run to run: bit-identical (test_fit_is_bit_exact_run_to_run).
    So no implementation can promise a per-patch MINIMUM of 0.999 here; what is asserted is the north-star figure on the
    mean (>= 0.999), the 1 % quantile >= 0.998, a floor of 0.99 on the minimum and every logged loss term within 6 %
    (+1e-3 absolute)."""
    from dvt.fit import FitEngine
    path = os.path.join(GOLD, "fit_headline_2000.npz")
    assert os.path.isfile(path), "tests/golden/fit_headline_2000.npz missing (tests/golden/make_fit_golden_headline.py)"
    cfg, z = _golden("headline_2000")
    feats, coords, init, idx, den, field, _ = _setup(cfg)
    assert int(idx.sum()) == int(z["idx_checksum"][0])
    eng = FitEngine(cfg["C"], cfg["h"], cfg["w"], cfg["bsz"], field.meta)
    eng.fit(den, field, feats.reshape(-1, cfg["C"]).cuda().contiguous(), coords.reshape(-1, 2).cuda().contiguous(), idx,
            graph_steps=20, lr=cfg["lr"], min_lr=cfg["min_lr"], warmup_iters=cfg["warmup_iters"],
            freeze_after=cfg["freeze_after"], weight_decay=cfg["weight_decay"], loss_scale=cfg["loss_scale"])
    denoised = eng.query(coords[-1:].cuda()).cpu()
    torch.cuda.synchronize()
    assert _L().device_error() == 0
    ref = torch.from_numpy(z["denoised_feats"].astype(np.float32))
    cos = F.cosine_similarity(denoised.reshape(-1, cfg["C"]), ref.reshape(-1, cfg["C"]), dim=-1)
    mean_c, q01, min_c = cos.mean().item(), cos.quantile(0.01).item(), cos.min().item()
    assert mean_c > 0.999, f"denoised_feats mean cosine after 2000 steps {mean_c}"
    assert q01 > 0.998, f"denoised_feats 1 % quantile of the per-patch cosine {q01}"
    assert min_c > 0.99, f"denoised_feats min cosine {min_c}"
    losses = eng.losses()
    worst = 0.0
    for row in z["logs"]:
        s = int(row[0])
        for j in range(5):
            ref_v, got_v = row[1 + j], losses[s, j]
            worst = max(worst, abs(got_v - ref_v) / (abs(ref_v) + 1e-3))
            assert abs(got_v - ref_v) <= 0.06 * abs(ref_v) + 1e-3, f"step {s} loss[{j}] {got_v} vs {ref_v}"
    tsum = float(eng.get_param("table", init["table"]).double().sum())
    assert abs(tsum - float(z["table_sum"][0])) <= 0.02 * float(z["table_sum"][1]) + 1e-3
    print(f"headline golden: cosine mean {mean_c:.6f} q01 {q01:.6f} min {min_c:.6f}, worst relative loss deviation {worst:.4f}")


def test_device_side_init_and_async_begin():
    """Per-image re-initialisation on the device (dvt_fit_init_params): right distributions, deterministic in the seed,
    different across seeds; a fit begun without host validation (validate=False) equals one begun with it; bad inputs are
    reported by begin(validate=True) and, for validate=False, by check()."""
    import dvt.models as DVT
    from dvt import _lib
    from dvt.fit import FitEngine
    from oracle import fit as OF
    C, h, w, V, bsz, L, T = 64, 6, 6, 4, 128, 6, 24
    field = DVT.NeuralFeatureField(feat_dim=C, n_levels=L)
    den = DVT.SingleImageDenoiser(h, w, C)
    eng = FitEngine(C, h, w, bsz, field.meta)
    eng.init_params(123)
    tab = eng.get_param("table", field.neural_field.params).cpu()
    assert tab.abs().max().item() <= 1e-4 and abs(tab.mean().item()) < 2e-6
    assert abs(tab.std().item() - 1e-4 / 3 ** 0.5) < 2e-6                       # U(-1e-4, 1e-4)
    w1 = eng.get_param("mlp.0.weight", field.mlp[0].weight).cpu()
    bound = 1.0 / (L * 8) ** 0.5
    assert w1.abs().max().item() <= bound and abs(w1.std().item() - bound / 3 ** 0.5) < 0.05 * bound
    G = eng.get_param("G", den.shared_artifacts).cpu()
    assert G.shape == den.shared_artifacts.shape and abs(G.std().item() - 0.02) < 2e-3 and abs(G.mean().item()) < 2e-3
    assert 2.5 < G.abs().max().item() / 0.02 < 6.0                               # a normal, not a uniform
    eng.init_params(123)
    assert torch.equal(eng.get_param("table", field.neural_field.params).cpu(), tab)
    eng.init_params(124)
    assert not torch.equal(eng.get_param("table", field.neural_field.params).cpu(), tab)
    # validate=False == validate=True
    feats, coords = OF.synthetic_bank(V, h, w, C, seed=0)
    bank, bco = feats.reshape(-1, C).cuda().contiguous(), coords.reshape(-1, 2).cuda().contiguous()
    idx = np.random.RandomState(0).randint(0, V * h * w, (T, bsz))
    hyper = dict(lr=0.01, min_lr=0.001, warmup_iters=3, freeze_after=0.5, weight_decay=1e-5, loss_scale=1024.0)
    outs = []
    for validate in (True, False):
        eng.init_params(7)
        eng.begin(bank, bco, idx, validate=validate, **hyper)
        eng.run(graph_steps=4)
        outs.append((eng.query(coords[-1:].cuda()).cpu(), eng.losses().copy()))
        eng.check()
    assert _min_cos(outs[0][0], outs[1][0]) > 0.99999 and np.allclose(outs[0][1], outs[1][1], rtol=1e-3, atol=1e-6)
    assert outs[0][1][-1, 0] < outs[0][1][4, 0]
    # losses_async == losses
    la = eng.losses_async()
    torch.cuda.synchronize()
    assert np.array_equal(la.numpy(), eng.losses())
    # bad inputs
    bad_co = bco.clone()
    bad_co[5, 0] = 1.5
    with pytest.raises(_lib.DvtError, match=r"coordinates should be in \[0, 1\]"):
        eng.begin(bank, bad_co, idx, **hyper)
    bad_idx = idx.copy()
    bad_idx[3, 3] = V * h * w + 9
    eng.begin(bank, bco, bad_idx, validate=False, **hyper)
    eng.run(4, graph_steps=0)                                                    # rows are clamped: no out-of-bounds read
    with pytest.raises(_lib.DvtError, match="out of range"):
        eng.check()
    eng.check()                                                                   # reported once, then cleared
    assert _lib.device_error() == 0


@pytest.mark.parametrize("n_levels,n", [(10, 1369), (6, 37), (16, 5)])
def test_encode_with_partial_last_warp(n_levels, n):
    """fit_query's encode with n * n_levels not a multiple of 8 (class-default 10 levels on a 37 x 37 map: the advisor's
    round-1 finding about full-mask shuffles after an early return) against the fp32 hash-grid op."""
    import dvt.models as DVT
    from dvt.fit import FitEngine
    C = 64
    field = DVT.NeuralFeatureField(feat_dim=C, n_levels=n_levels).cuda()
    with torch.no_grad():
        field.neural_field.params.uniform_(-1, 1, generator=None)
    den = DVT.SingleImageDenoiser(4, 4, C).cuda()
    eng = FitEngine(C, 4, 4, 64, field.meta)
    eng.load_modules(den, field)
    co = torch.rand(n, 2, device="cuda", generator=torch.Generator(device="cuda").manual_seed(n))
    got = eng.query(co)
    with torch.no_grad():
        ref = field(co)                       # hash-grid op (fp32 kernel) + torch Linear layers
    torch.cuda.synchronize()
    assert (got - ref).abs().max().item() < 2e-3 * max(1.0, ref.abs().max().item())
    assert _L().device_error() == 0


def test_sweep_kernels_agree(monkeypatch):
    """The TMA-staged dense Adam sweep (`fit_adam_table_tma_kernel`, the default of the pipelined schedule) against the
    plain-load kernel: (i) one sweep from the same state is BIT-identical (same adam1() arithmetic), incl. a ragged last
    chunk; (ii) whole fits with either kernel agree within the tolerance below."""
    import dvt.models as DVT
    from dvt.fit import FitEngine
    # (i) 10 levels on purpose: 1 740 464 entries = 3399 chunks of 512 + a ragged one
    C, h, w, bsz, L, T = 64, 6, 6, 128, 10, 8
    field = DVT.NeuralFeatureField(feat_dim=C, n_levels=L)
    assert (field.meta.n_params // 8) % 512 != 0
    g = torch.Generator(device="cuda").manual_seed(0)
    bank = torch.randn(4 * h * w, C, device="cuda", generator=g)
    co = torch.rand(4 * h * w, 2, device="cuda", generator=g)
    idx = np.random.RandomState(0).randint(0, 4 * h * w, (T, bsz))
    hyper = dict(lr=0.01, min_lr=0.001, warmup_iters=0, freeze_after=0.5, weight_decay=0.37, loss_scale=1024.0)
    outs = []
    for ctas in (7, -7, 0):          # TMA-staged on 7 CTAs, plain loads on 7 CTAs, plain loads on the full grid
        monkeypatch.setenv("DVT_FIT_SWEEP_TMA", "1" if ctas > 0 else "0")
        eng = FitEngine(C, h, w, bsz, field.meta)
        eng.init_params(5)
        eng.begin(bank, co, idx, **hyper)
        eng.sweep_once(ctas)
        outs.append(eng.get_param("table.next", field.neural_field.params).cpu())
        torch.cuda.synchronize()
        assert _L().device_error() == 0
        start = eng.get_param("table", field.neural_field.params).cpu()
    assert not torch.equal(outs[0], start), "the sweep must have changed the table (weight decay 0.37, lr 0.01)"
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[1], outs[2])
    # (ii) whole fits
    cfg, z = _golden("hashed_L16")
    res = []
    for tma in ("1", "0"):
        monkeypatch.setenv("DVT_FIT_SWEEP_TMA", tma)     # read by dvt_fit_create
        monkeypatch.setenv("DVT_FIT_SWEEP_CTAS", "5,3")
        feats, coords, init, idx2, den, fld, _ = _setup(cfg)
        eng = FitEngine(cfg["C"], cfg["h"], cfg["w"], cfg["bsz"], fld.meta)
        eng.fit(den, fld, feats.reshape(-1, cfg["C"]).cuda().contiguous(), coords.reshape(-1, 2).cuda().contiguous(), idx2,
                graph_steps=5, lr=cfg["lr"], min_lr=cfg["min_lr"], warmup_iters=cfg["warmup_iters"],
                freeze_after=cfg["freeze_after"], weight_decay=cfg["weight_decay"], loss_scale=cfg["loss_scale"])
        torch.cuda.synchronize()
        assert _L().device_error() == 0
        res.append((eng.get_param("table", init["table"]).cpu() - init["table"], eng.losses().copy(),
                    eng.query(coords[-1:].cuda()).cpu()))
    (ta, la, qa), (tb, lb, qb) = res
    assert F.cosine_similarity(ta.flatten().double(), tb.flatten().double(), dim=0).item() > 0.9999
    assert np.allclose(la, lb, rtol=1e-3, atol=1e-5)
    assert _min_cos(qa, torch.from_numpy(z["denoised_feats"])) > 0.999
