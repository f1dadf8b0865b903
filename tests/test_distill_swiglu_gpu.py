"""Stage-3 distillation of the SwiGLU backbones (ViT-g/14, timm SwiGLUPacked MLP) on the GPU: the fused SwiGLU-backward
data-gradient GEMM and the SwiGLU forward against torch, every parameter gradient of the ViT against autograd through the
fp32 oracle (oracle/vit.py `embed` / `block`), the training forward against the inference forward, weights after an
optimiser step, gradient checkpointing, a short AdamW run against torch.optim.AdamW on the oracle, the drop-in command line
on a ViT-g tag, and one full-size ViT-g step.
Tolerances as tests/test_distill_gpu.py: bf16 tensor-core GEMMs / attention with fp32 accumulation against fp32 references ->
cosine >= 0.99 and norm ratio 0.95-1.05 on every parameter gradient."""
import contextlib
import os
import re
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G14 = "vit_giant_patch14_dinov2.lvd142m"
G14_REG = "vit_giant_patch14_reg4_dinov2.lvd142m"
NARROW = dict(embed=384, heads=6, mlp=2048)      # the ViT-g block layout (SwiGLU, LayerScale) at ViT-S width


def _cos(a, b):
    return F.cosine_similarity(a.flatten().double(), b.flatten().double(), dim=0).item()


def _dev_ok():
    from dvt import _lib
    torch.cuda.synchronize()
    assert _lib.device_error() == 0


@contextlib.contextmanager
def _impl(name):
    from dvt import _lib
    _lib.check(_lib.lib().dvt_set_debug_impl(1 if name == "simt" else 0))
    try:
        yield
    finally:
        _lib.check(_lib.lib().dvt_set_debug_impl(-1))


# ---------------------------------------------------------------------------------------------------------------------
# kernel units
# ---------------------------------------------------------------------------------------------------------------------
def _swiglu_bwd_ref(dy, w, hpre):
    """fp32 composite: dh = dy @ w, then the SwiGLU backward on hpre = [g | u]."""
    Hh = w.shape[1]
    dh = dy.float() @ w.float()
    g, u = hpre.float()[:, :Hh], hpre.float()[:, Hh:]
    s = torch.sigmoid(g)
    silu = g * s
    return dh * u * (s + silu * (1 - s)), dh * silu


def _check_halves(got, ref_g, ref_u):
    Hh = ref_g.shape[1]
    for half, ref in ((got[:, :Hh].float(), ref_g), (got[:, Hh:].float(), ref_u)):
        assert torch.isfinite(half).all()
        err = (half - ref).abs().max().item()
        assert err <= 1e-2 * ref.abs().max().item(), (err, ref.abs().max().item())
        assert _cos(half, ref) >= 0.9999, _cos(half, ref)


# (M, C, Hh, row pitch of W2): Hh = 1000 ends in a partial tile; Hh = 1002 (W2 padded to a 16-byte row pitch) is not a
# multiple of 4 and takes the scalar epilogue everywhere
SHAPES = [(333, 384, 1024, None), (2740, 1536, 4096, None), (333, 384, 1000, None), (333, 384, 1002, 1008)]


@pytest.mark.parametrize("impl", ["tc", "simt"])
@pytest.mark.parametrize("M,C,Hh,ldw", SHAPES, ids=[f"{m}x{c}x{h}" + ("pad" if p else "") for m, c, h, p in SHAPES])
def test_dgrad_swiglu_matches_torch(impl, M, C, Hh, ldw):
    from dvt import train_ops
    g = torch.Generator(device="cuda").manual_seed(M + Hh)
    dy = torch.randn(M, C, device="cuda", generator=g).bfloat16()
    wfull = (torch.randn(C, ldw or Hh, device="cuda", generator=g) / 32).bfloat16()
    w = wfull[:, :Hh]
    hpre = (2 * torch.randn(M, 2 * Hh, device="cuda", generator=g)).bfloat16()
    with _impl(impl):
        got = train_ops.dgrad_swiglu(dy, w, hpre)
        again = train_ops.dgrad_swiglu(dy, w, hpre)
        _dev_ok()
    assert got.shape == (M, 2 * Hh) and got.dtype == torch.bfloat16
    _check_halves(got, *_swiglu_bwd_ref(dy, w, hpre))
    assert torch.equal(got, again)                      # plain stores, no split-K: bit-identical repeats


@pytest.mark.parametrize("impl", ["tc", "simt"])
def test_dgrad_swiglu_extreme_preactivations(impl):
    """g at +-30, +-88 and +-1e4 (exp(-g) overflows at -88 and -1e4): finite, and equal to torch's F.silu autograd."""
    from dvt import train_ops
    M, C, Hh = 256, 384, 512
    g = torch.Generator(device="cuda").manual_seed(11)
    dy = torch.randn(M, C, device="cuda", generator=g).bfloat16()
    w = (torch.randn(C, Hh, device="cuda", generator=g) / 32).bfloat16()
    vals = torch.tensor([30.0, -30.0, 88.0, -88.0, 1e4, -1e4, 0.0, 1.5], device="cuda")
    gate = vals[torch.randint(0, len(vals), (M, Hh), device="cuda", generator=g)]
    up = torch.randn(M, Hh, device="cuda", generator=g)
    hpre = torch.cat([gate, up], 1).bfloat16().contiguous()
    with _impl(impl):
        got = train_ops.dgrad_swiglu(dy, w, hpre)
        _dev_ok()
    gt = hpre[:, :Hh].float().requires_grad_(True)
    ut = hpre[:, Hh:].float().requires_grad_(True)
    dh = dy.float() @ w.float()
    (F.silu(gt) * ut).backward(dh)
    _check_halves(got, gt.grad, ut.grad)


def test_swiglu_forward_within_one_ulp():
    from dvt import train_ops
    g = torch.Generator(device="cuda").manual_seed(5)
    M, Hh = 1000, 4096
    hpre = (3 * torch.randn(M, 2 * Hh, device="cuda", generator=g)).bfloat16()
    got = train_ops.swiglu(hpre)
    _dev_ok()
    ref = (F.silu(hpre[:, :Hh].float()) * hpre[:, Hh:].float()).bfloat16().float()
    ulp = torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(1e-30))) - 7)
    assert ((got.float() - ref).abs() <= ulp).all(), (got.float() - ref).abs().max().item()


# ---------------------------------------------------------------------------------------------------------------------
# the whole ViT against the oracle
# ---------------------------------------------------------------------------------------------------------------------
def _pair(ident, stride, over=None, seed=0):
    """(wrapper on cuda with oracle weights, oracle config, oracle state dict) for `ident` with the arch fields in `over`
    replaced.  The wrapper is built with the replaced arch, so a shallow ViT-g never allocates the 40-block model."""
    import dvt.models as DVT
    from dvt.models import vit_wrapper as VW
    from oracle import vit as OV
    a = {**VW.ARCHS[ident], **(over or {})}
    P = int(re.search(r"patch(\d+)", ident).group(1))
    cfg = OV.ViTConfig(a["embed"], a["depth"], a["heads"], P, a["img"], a["mlp"], a["swiglu"], a["ls"], a["reg"],
                       a["no_embed_class"])
    sd = OV.random_state_dict(cfg, seed=seed)
    old = VW.ARCHS[ident]
    VW.ARCHS[ident] = a
    try:
        w = DVT.PretrainedViTWrapper(ident, stride=stride, allow_random_init=True)
    finally:
        VW.ARCHS[ident] = old
    w.model.load_state_dict(sd, strict=True)
    return w.cuda(), cfg, sd


def _oracle_loss(params, cfg, x, target, stride):
    """main_distillation.py:233-238 on the oracle forward (last layer, final norm, prefix stripped)."""
    from oracle import vit as OV
    B, _, H, W = x.shape
    h, w = OV.feat_size(cfg, H, W, stride)
    t = OV.embed(params, cfg, x, stride)
    for i in range(cfg.depth):
        t = OV.block(t, params, i, cfg)
    t = F.layer_norm(t, (cfg.embed_dim,), params["norm.weight"], params["norm.bias"], cfg.ln_eps)
    feat = t[:, cfg.num_prefix:].reshape(B, h, w, -1)
    l2 = F.mse_loss(feat, target)
    cs = 1 - F.cosine_similarity(feat, target, dim=-1).mean()
    return l2 + cs, feat


def _oracle_grads(sd, cfg, x, target, stride):
    params = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    loss, feat = _oracle_loss(params, cfg, x, target, stride)
    loss.backward()
    return loss.item(), {k: p.grad for k, p in params.items()}, feat.detach()


def _our_grads(w, x, target):
    from dvt import train_ops
    w.set_trainable(True)
    for p in w.parameters():
        p.grad = None
    pred = w.get_intermediate_layers(x.cuda())[0].permute(0, 2, 3, 1)
    loss, _, _ = train_ops.denoise_loss(pred, target.cuda())
    loss.backward()
    _dev_ok()
    return loss.item(), {k[len("model."):]: p.grad.detach().cpu() for k, p in w.named_parameters()}, pred.detach().cpu()


CASES = {
    "vitg14-depth2": dict(ident=G14, stride=14, over=dict(depth=2, img=98), hw=(98, 112)),
    "vitg14-reg4-stride7": dict(ident=G14_REG, stride=7, over=dict(depth=2, img=98), hw=(70, 70)),
    "swiglu-narrow-full-depth": dict(ident=G14, stride=14, over=dict(NARROW, depth=12, img=98), hw=(98, 98)),
}


@pytest.mark.parametrize("case", list(CASES))
def test_swiglu_vit_gradients_match_oracle(case):
    """Loss and the gradient of EVERY backbone parameter against autograd through the fp32 oracle (LayerScale drawn from
    U(0.5, 1.5), so every branch matters)."""
    c = CASES[case]
    w, cfg, sd = _pair(c["ident"], c["stride"], c["over"], seed=3)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 3, *c["hw"], generator=g)
    from oracle import vit as OV
    h, wd = OV.feat_size(cfg, c["hw"][0], c["hw"][1], c["stride"])
    target = torch.randn(2, h, wd, cfg.embed_dim, generator=g)
    r_loss, r_grads, r_feat = _oracle_grads(sd, cfg, x, target, c["stride"])
    loss, grads, feat = _our_grads(w, x, target)
    assert F.cosine_similarity(feat.reshape(-1, cfg.embed_dim), r_feat.reshape(-1, cfg.embed_dim), dim=-1).min().item() > 0.99
    assert abs(loss - r_loss) < 2e-2 * abs(r_loss), (loss, r_loss)
    assert set(grads) == set(r_grads)
    for name, gr in grads.items():
        c_ = _cos(gr, r_grads[name])
        assert c_ > 0.99, f"{name}: gradient cosine {c_}"
        ratio = gr.norm().item() / (r_grads[name].norm().item() + 1e-12)
        assert 0.95 < ratio < 1.05, f"{name}: gradient norm ratio {ratio}"


# ---------------------------------------------------------------------------------------------------------------------
# forward and weight handling
# ---------------------------------------------------------------------------------------------------------------------
def test_vitg_training_forward_equals_inference_forward():
    w, cfg, _ = _pair(G14, 14, dict(depth=2, img=98))
    x = torch.randn(2, 3, 112, 98, generator=torch.Generator().manual_seed(1)).cuda()
    ref = w.get_intermediate_layers(x)[0]
    assert ref.grad_fn is None
    w.set_trainable(True)
    got = w.get_intermediate_layers(x)[0]
    _dev_ok()
    assert got.grad_fn is not None and got.shape == ref.shape
    C = cfg.embed_dim
    flat = lambda t: t.detach().permute(0, 2, 3, 1).reshape(-1, C)  # noqa: E731
    assert F.cosine_similarity(flat(got), flat(ref), dim=-1).min().item() > 0.9999


def test_swiglu_inference_after_optimiser_step_uses_the_new_weights():
    from dvt import train_ops
    from dvt.optim import FusedAdamW
    from dvt.models import vit_wrapper as VW
    w, cfg, _ = _pair(G14, 14, dict(NARROW, depth=3, img=98))
    x = torch.randn(2, 3, 98, 98, generator=torch.Generator().manual_seed(2)).cuda()
    before = w.get_intermediate_layers(x)[0].clone()
    w.set_trainable(True)
    opt = FusedAdamW(w.parameters(), lr=1e-3, weight_decay=1e-5)
    loss, _, _ = train_ops.denoise_loss(w.get_intermediate_layers(x)[0].permute(0, 2, 3, 1), torch.zeros(2, 7, 7, 384).cuda())
    opt.zero_grad()
    loss.backward()
    opt.step()
    w.set_trainable(False)
    after = w.get_intermediate_layers(x)[0]
    fresh = VW.B200VisionTransformer(G14, 14, w.model.arch)
    fresh.load_state_dict({k[len("model."):]: v.detach().cpu().clone() for k, v in w.state_dict().items()}, strict=True)
    fresh = fresh.cuda()
    ref = fresh.forward_intermediates(x, [cfg.depth - 1], norm=True, output_fmt="NCHW", intermediates_only=True)[0]
    _dev_ok()
    assert not torch.equal(after, before)
    assert (after - ref).abs().max().item() < 1e-5 * ref.abs().max().item()


def test_swiglu_gradient_checkpointing_same_result_less_memory():
    w, cfg, _ = _pair(G14, 14, dict(NARROW, depth=12, img=224))
    g = torch.Generator().manual_seed(6)
    x = torch.randn(8, 3, 224, 224, generator=g)
    target = torch.randn(8, 16, 16, cfg.embed_dim, generator=g)
    runs = []
    for ckpt in (False, True):
        w.model.set_grad_checkpointing(ckpt)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        loss, grads, feat = _our_grads(w, x, target)
        runs.append((loss, grads, torch.cuda.max_memory_allocated() - base, feat))
    (l0, g0, m0, f0), (l1, g1, m1, f1) = runs
    assert torch.equal(f0, f1) and abs(l0 - l1) < 1e-6 * abs(l0)
    for k in g0:
        assert _cos(g0[k], g1[k]) > 0.9999, k
    assert m1 < 0.6 * m0, (m0, m1)


# ---------------------------------------------------------------------------------------------------------------------
# short run against the oracle loop
# ---------------------------------------------------------------------------------------------------------------------
def test_swiglu_training_run_matches_oracle():
    """20 AdamW steps (warm-up + cosine schedule): FusedAdamW on the CUDA path against torch.optim.AdamW on the fp32 oracle."""
    from dvt import train_ops
    from dvt.optim import FusedAdamW
    from dvt.utils import misc
    T, B = 20, 2
    w, cfg, sd = _pair(G14, 14, dict(NARROW, depth=3, img=98), seed=8)
    g = torch.Generator().manual_seed(9)
    imgs = torch.randn(4, 3, 98, 98, generator=g)
    targets = torch.randn(4, 7, 7, cfg.embed_dim, generator=g)
    batches = [torch.randint(0, 4, (B,), generator=g) for _ in range(T)]
    sched = dict(base_value=1e-3, final_value=1e-5, total_iters=T, warmup_iters=int(T * 0.15), start_warmup_value=0)
    params = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    ropt = torch.optim.AdamW(list(params.values()), betas=(0.9, 0.999), weight_decay=1e-5)
    ref_logs = []
    for s, ids in enumerate(batches):
        for grp in ropt.param_groups:
            grp["lr"] = misc.cosine_schedule(s, **sched)
        loss, _ = _oracle_loss(params, cfg, imgs[ids], targets[ids], 14)
        ropt.zero_grad()
        loss.backward()
        ropt.step()
        ref_logs.append(loss.item())
    w.set_trainable(True)
    opt = FusedAdamW(w.parameters(), betas=(0.9, 0.999), weight_decay=1e-5)
    logs = []
    for s, ids in enumerate(batches):
        misc.apply_optim_scheduler(opt, misc.cosine_schedule(s, **sched))
        pred = w.get_intermediate_layers(imgs[ids].cuda())[0].permute(0, 2, 3, 1)
        loss, _, _ = train_ops.denoise_loss(pred, targets[ids].cuda())
        opt.zero_grad()
        loss.backward()
        opt.step()
        logs.append(loss.item())
    _dev_ok()
    logs, ref_logs = np.array(logs), np.array(ref_logs)
    assert np.allclose(logs, ref_logs, rtol=0.03, atol=2e-3), np.abs(logs - ref_logs).max()
    assert logs[-1] < logs[0]
    got = {k[len("model."):]: v.detach().cpu() for k, v in w.state_dict().items()}
    C = cfg.embed_dim
    for k, v in params.items():
        upd_ref, upd_got = v.detach() - sd[k], got[k] - sd[k]
        if k.endswith("attn.qkv.bias"):
            # softmax is invariant to a shift of all keys: the exact k-bias gradient is zero, what Adam normalises there is
            # rounding noise -- compare the q and v thirds only
            keep = torch.cat([torch.arange(0, C), torch.arange(2 * C, 3 * C)])
            upd_ref, upd_got = upd_ref[keep], upd_got[keep]
        assert _cos(upd_got, upd_ref) > 0.97, f"{k}: update cosine {_cos(upd_got, upd_ref)}"


# ---------------------------------------------------------------------------------------------------------------------
# command line and the full-size model
# ---------------------------------------------------------------------------------------------------------------------
def test_stage3_cli_trains_vitg_with_checkpointing(tmp_path, capsys, monkeypatch):
    """main_distillation.py on the ViT-g/14 reg4 tag at stride 7 with --grad_checkpointing (two blocks, so that a checkpoint
    stays small), the teacher a Denoiser(feat_dim=1536) in the stage-2 checkpoint layout: the loss falls, the checkpoint loads
    strictly into a fresh wrapper, `--resume` continues."""
    from PIL import Image
    import dvt.models as DVT
    from dvt.models import vit_wrapper as VW
    sys.path.insert(0, ROOT)
    import main_distillation as M
    ident = G14_REG
    monkeypatch.setitem(VW.ARCHS, ident, {**VW.ARCHS[ident], "depth": 2})
    half = np.random.RandomState(0).randint(0, 255, (70, 35, 3), dtype=np.uint8)
    img = np.ascontiguousarray(np.concatenate([half, half[:, ::-1]], axis=1))
    for i in range(8):
        d = tmp_path / "data" / f"class{i % 2}"
        d.mkdir(parents=True, exist_ok=True)
        Image.fromarray(img).save(d / f"{i}.png")
    torch.manual_seed(0)
    vit = VW.B200VisionTransformer(ident, 14, VW.ARCHS[ident])
    for blk in vit.blocks:
        blk.ls1.gamma.data.fill_(1.0)
        blk.ls2.gamma.data.fill_(1.0)
    wdir = tmp_path / "weights"
    wdir.mkdir()
    torch.save(vit.state_dict(), wdir / f"{ident}.pth")
    monkeypatch.setenv("DVT_WEIGHTS_DIR", str(wdir))
    den = DVT.Denoiser(9, 9, 1536, vit=None, num_blocks=1)
    torch.save({"denoiser": den.state_dict(), "optimizer": {}, "step": 0}, tmp_path / "denoiser.pth")
    argv = ["--model", ident, "--denoiser_ckpt", str(tmp_path / "denoiser.pth"), "--input_size", "70", "--stride_size", "7",
            "--data_root", str(tmp_path / "data"), "--batch_size", "4", "--num_iterations", "12", "--blr", "0.002",
            "--output_root", str(tmp_path / "work"), "--run_name", "t", "--save_freq", "1000", "--num_workers", "0",
            "--log_freq", "3", "--grad_checkpointing"]
    M.main(M.get_args(argv))
    out = capsys.readouterr().out
    assert "Enable gradient checkpointing" in out
    vals = [float(ln.split("loss: ")[1].split()[0]) for ln in out.splitlines() if ln.startswith("Train [")]
    assert len(vals) >= 3 and vals[-1] < vals[0], vals
    ck_dir = tmp_path / "work" / "denosing-vit" / "t" / "checkpoints"
    assert sorted(os.listdir(ck_dir)) == ["ckpt_000000.pth", "ckpt_000011.pth", "latest.pth"]
    ck = torch.load(str(ck_dir / "latest.pth"), map_location="cpu")
    assert ck["step"] == 11 and "model.blocks.1.mlp.fc2.weight" in ck["model"]
    assert tuple(ck["model"]["model.blocks.1.mlp.fc2.weight"].shape) == (1536, 4096)
    fresh = DVT.PretrainedViTWrapper(ident, stride=7, allow_random_init=True)
    fresh.load_state_dict(ck["model"], strict=True)
    os.remove(ck_dir / "ckpt_000000.pth")
    i = argv.index("--num_iterations")
    M.main(M.get_args(argv[:i + 1] + ["14"] + argv[i + 2:] + ["--resume", str(ck_dir / "latest.pth")]))
    out2 = capsys.readouterr().out
    assert "Resumed from" in out2 and "at step 12" in out2 and os.path.isfile(ck_dir / "ckpt_000013.pth")


def test_vitg_full_size_step_with_checkpointing():
    """One full-depth ViT-g/14 step at 518 x 518, batch 2, gradient checkpointing, FusedAdamW: a finite loss, no device
    error; prints the peak memory."""
    import dvt.models as DVT
    from dvt import train_ops
    from dvt.optim import FusedAdamW
    with torch.device("cuda"):
        w = DVT.PretrainedViTWrapper(G14, stride=14, allow_random_init=True)
    w = w.cuda()
    w.set_trainable(True)
    w.model.set_grad_checkpointing(True)
    opt = FusedAdamW(w.parameters(), lr=1e-5, weight_decay=1e-5)
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(2, 3, 518, 518, device="cuda", generator=g)
    target = torch.randn(2, 37, 37, 1536, device="cuda", generator=g)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    pred = w.get_intermediate_layers(x)[0].permute(0, 2, 3, 1)
    loss, _, _ = train_ops.denoise_loss(pred, target)
    opt.zero_grad()
    loss.backward()
    opt.step()
    _dev_ok()
    assert np.isfinite(loss.item())
    assert all(torch.isfinite(p).all() for p in w.parameters())
    print(f"ViT-g/14 518x518 batch 2 checkpointed step: loss {loss.item():.4f}, peak memory "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
