"""Stage-3 distillation on the GPU (reference main_distillation.py): the new kernels against torch fp32, the gradients of the
whole ViT (patch embedding, LayerScale blocks, final norm + prefix strip, position / cls / register tokens) against autograd
through the CPU oracle (oracle/vit.py `embed` / `block`, fp32), the training forward against the inference forward, weight
handling after optimiser steps, gradient checkpointing, a short AdamW run against torch.optim.AdamW on the oracle, and the
drop-in command line end to end.
Tolerances as tests/test_train_gpu.py: bf16 tensor-core GEMMs / attention with fp32 accumulation against fp32 references ->
cosine >= 0.99 and norm ratio 0.95-1.05 on every parameter gradient, fp32 elementwise kernels to ~1e-5 relative."""
import os
import re
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cos(a, b):
    return F.cosine_similarity(a.flatten().double(), b.flatten().double(), dim=0).item()


def _dev_ok():
    from dvt import _lib
    torch.cuda.synchronize()
    assert _lib.device_error() == 0


# ---------------------------------------------------------------------------------------------------------------------
# kernel units
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,C", [(1370, 768), (333, 384)])
@pytest.mark.parametrize("with_gamma", [True, False], ids=["layerscale", "plain"])
def test_layerscale_backward(rows, C, with_gamma):
    from dvt import train_ops
    g = torch.Generator(device="cuda").manual_seed(rows + C)
    dx = torch.randn(rows, C, device="cuda", generator=g)
    branch = torch.randn(rows, C, device="cuda", generator=g).bfloat16()
    gamma = (0.5 + torch.rand(C, device="cuda", generator=g)) if with_gamma else None
    dbr, dbias, dgamma = train_ops.layerscale_bwd(dx, branch if with_gamma else None, gamma)
    dbr2, dbias2, dgamma2 = train_ops.layerscale_bwd(dx, branch if with_gamma else None, gamma)
    _dev_ok()
    gd = dx.double() * (gamma.double() if with_gamma else 1.0)
    assert torch.equal(dbr, gd.float().bfloat16())
    assert (dbias.double() - gd.sum(0)).abs().max().item() < 1e-5 * gd.abs().sum(0).max().item()
    if with_gamma:
        ref = (dx.double() * branch.double()).sum(0)
        assert (dgamma.double() - ref).abs().max().item() < 1e-5 * (dx.double() * branch.double()).abs().sum(0).max().item()
        assert torch.equal(dgamma, dgamma2)
    else:
        assert dgamma is None
    assert torch.equal(dbias, dbias2) and torch.equal(dbr, dbr2)        # fixed-order sums: bit-identical repeats


@pytest.mark.parametrize("prefix", [1, 5])
def test_vit_embed_backward(prefix):
    from dvt import train_ops
    g = torch.Generator(device="cuda").manual_seed(prefix)
    B, np_, C = 3, 81, 384
    ntok = prefix + np_
    dx0 = torch.randn(B * ntok, C, device="cuda", generator=g)
    dpatch, dpos, dprefix, dbias = train_ops.vit_embed_bwd(dx0, B, prefix)
    again = train_ops.vit_embed_bwd(dx0, B, prefix)
    _dev_ok()
    t = dx0.view(B, ntok, C).double()
    assert torch.equal(dpatch, dx0.view(B, ntok, C)[:, prefix:].reshape(-1, C).bfloat16())
    assert (dpos.double() - t[:, prefix:].sum(0)).abs().max().item() < 1e-5
    assert (dprefix.double() - t[:, :prefix].sum(0)).abs().max().item() < 1e-5
    assert (dbias.double() - t[:, prefix:].sum((0, 1))).abs().max().item() < 1e-4
    assert all(torch.equal(a, b) for a, b in zip((dpatch, dpos, dprefix, dbias), again))


@pytest.mark.parametrize("prefix,C", [(1, 384), (5, 768)])
def test_grouped_layernorm_backward(prefix, C):
    from dvt import train_ops
    g = torch.Generator(device="cuda").manual_seed(C)
    B, np_ = 3, 49
    ntok = prefix + np_
    x = (torch.randn(B * ntok, C, device="cuda", generator=g) * 2 + 0.3).requires_grad_(True)
    w = (1 + 0.2 * torch.randn(C, device="cuda", generator=g)).requires_grad_(True)
    b = (0.1 * torch.randn(C, device="cuda", generator=g)).requires_grad_(True)
    dy = torch.randn(B * np_, C, device="cuda", generator=g)
    y = F.layer_norm(x, (C,), w, b, 1e-6).view(B, ntok, C)[:, prefix:].reshape(-1, C)
    y.backward(dy)
    acc0 = torch.randn(B * ntok, C, device="cuda", generator=g)
    acc = acc0.clone()
    dg, db = train_ops.layernorm_bwd_grouped_(acc, x.detach(), w.detach(), dy, ntok, prefix)
    acc2 = acc0.clone()
    dg2, db2 = train_ops.layernorm_bwd_grouped_(acc2, x.detach(), w.detach(), dy, ntok, prefix)
    _dev_ok()
    assert (acc - acc0 - x.grad).abs().max().item() < 2e-4 * max(1.0, x.grad.abs().max().item())
    assert torch.equal(acc.view(B, ntok, C)[:, :prefix], acc0.view(B, ntok, C)[:, :prefix])   # prefix rows untouched
    assert (dg - w.grad).abs().max().item() < 2e-4 * w.grad.abs().max().item() + 1e-4
    assert (db - b.grad).abs().max().item() < 2e-4 * b.grad.abs().max().item() + 1e-4
    assert torch.equal(dg, dg2) and torch.equal(db, db2) and torch.equal(acc, acc2)


@pytest.mark.parametrize("impl", ["tc", "simt"])
@pytest.mark.parametrize("with_gamma", [True, False], ids=["layerscale", "plain"])
def test_residual_gemm_keeps_the_branch(impl, with_gamma):
    from dvt import _lib, ops
    g = torch.Generator(device="cuda").manual_seed(7)
    M, N, K = 333, 384, 256
    a = torch.randn(M, K, device="cuda", generator=g).bfloat16()
    w = (torch.randn(N, K, device="cuda", generator=g) / 16).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g)
    gamma = (0.5 + torch.rand(N, device="cuda", generator=g)) if with_gamma else None
    x0 = torch.randn(M, N, device="cuda", generator=g)
    _lib.check(_lib.lib().dvt_set_debug_impl(1 if impl == "simt" else 0))
    try:
        x1 = ops.gemm_tn_residual_(x0.clone(), a, w, bias, gamma)
        branch = torch.empty(M, N, device="cuda", dtype=torch.bfloat16)
        x2 = ops.gemm_tn_residual_(x0.clone(), a, w, bias, gamma, branch)
        x3 = ops.gemm_tn_residual_(x0.clone(), a, w, bias, gamma, None)
        _dev_ok()
    finally:
        _lib.check(_lib.lib().dvt_set_debug_impl(-1))
    assert torch.equal(x1, x2) and torch.equal(x1, x3)
    ref = a.float() @ w.float().t() + bias
    assert (branch.float() - ref).abs().max().item() < 1e-2 * ref.abs().max().item()


# ---------------------------------------------------------------------------------------------------------------------
# the whole ViT against the oracle
# ---------------------------------------------------------------------------------------------------------------------
def _pair(ident, stride, depth=None, img=None, seed=0):
    """(wrapper on cuda with oracle weights, oracle config, oracle state dict) -- optionally a shallower / smaller-grid
    variant of the architecture."""
    import dvt.models as DVT
    from dvt.models import vit_wrapper as VW
    from oracle import vit as OV
    a = dict(VW.ARCHS[ident])
    if depth:
        a["depth"] = depth
    if img:
        a["img"] = img
    P = int(re.search(r"patch(\d+)", ident).group(1))
    cfg = OV.ViTConfig(a["embed"], a["depth"], a["heads"], P, a["img"], a["mlp"], a["swiglu"], a["ls"], a["reg"],
                       a["no_embed_class"])
    sd = OV.random_state_dict(cfg, seed=seed)
    w = DVT.PretrainedViTWrapper(ident, stride=stride, allow_random_init=True)
    w.model = VW.B200VisionTransformer(ident, P, a)
    w.model.patch_embed.proj.stride = [stride, stride]
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
    "dinov2-s14": dict(ident="vit_small_patch14_dinov2.lvd142m", stride=14, depth=3, img=98, hw=(98, 112)),
    "reg4-stride7": dict(ident="vit_small_patch14_reg4_dinov2.lvd142m", stride=7, depth=3, img=98, hw=(70, 70)),
    "dino-s16-resampled": dict(ident="vit_small_patch16_224.dino", stride=16, depth=3, img=None, hw=(96, 112)),
    "dinov2-s14-full-depth": dict(ident="vit_small_patch14_dinov2.lvd142m", stride=14, depth=None, img=None, hw=(98, 98)),
}


@pytest.mark.parametrize("case", list(CASES))
def test_vit_gradients_match_oracle(case):
    """Loss and the gradient of EVERY backbone parameter against autograd through the fp32 oracle.  The full-depth
    case runs 12 LayerScale blocks (gamma drawn from U(0.5, 1.5), far larger than DINOv2's 1e-5, so every branch matters)."""
    c = CASES[case]
    w, cfg, sd = _pair(c["ident"], c["stride"], c["depth"], c["img"], seed=3)
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
@pytest.mark.parametrize("norm,reshape", [(True, True), (False, False)])
def test_training_forward_equals_inference_forward(norm, reshape):
    w, cfg, _ = _pair("vit_small_patch14_reg4_dinov2.lvd142m", 14, img=98)
    x = torch.randn(2, 3, 112, 98, generator=torch.Generator().manual_seed(1)).cuda()
    ref = w.get_intermediate_layers(x, reshape=reshape, norm=norm)[0]
    assert ref.grad_fn is None                   # not trainable: the inference path, even with grad enabled
    w.set_trainable(True)
    got = w.get_intermediate_layers(x, reshape=reshape, norm=norm)[0]
    _dev_ok()
    assert got.grad_fn is not None and got.shape == ref.shape
    C = cfg.embed_dim
    flat = (lambda t: t.permute(0, 2, 3, 1).reshape(-1, C)) if reshape else (lambda t: t.reshape(-1, C))
    assert F.cosine_similarity(flat(got.detach()), flat(ref), dim=-1).min().item() > 0.9999
    with torch.no_grad():
        assert w.get_intermediate_layers(x, reshape=reshape, norm=norm)[0].grad_fn is None


def test_inference_after_optimiser_step_uses_the_new_weights():
    import dvt.models as DVT
    from dvt import train_ops
    from dvt.optim import FusedAdamW
    from dvt.models import vit_wrapper as VW
    w, cfg, _ = _pair("vit_small_patch14_dinov2.lvd142m", 14, depth=3, img=98)
    x = torch.randn(2, 3, 98, 98, generator=torch.Generator().manual_seed(2)).cuda()
    before = w.get_intermediate_layers(x)[0].clone()           # fills the handle's bf16 copies and position tables
    w.set_trainable(True)
    opt = FusedAdamW(w.parameters(), lr=1e-3, weight_decay=1e-5)
    loss, _, _ = train_ops.denoise_loss(w.get_intermediate_layers(x)[0].permute(0, 2, 3, 1), torch.zeros(2, 7, 7, 384).cuda())
    opt.zero_grad()
    loss.backward()
    opt.step()
    w.set_trainable(False)
    after = w.get_intermediate_layers(x)[0]
    fresh = DVT.PretrainedViTWrapper("vit_small_patch14_dinov2.lvd142m", stride=14, allow_random_init=True)
    fresh.model = VW.B200VisionTransformer("vit_small_patch14_dinov2.lvd142m", 14, w.model.arch)
    fresh.load_state_dict({k: v.detach().cpu().clone() for k, v in w.state_dict().items()}, strict=True)
    ref = fresh.cuda().get_intermediate_layers(x)[0]
    _dev_ok()
    assert not torch.equal(after, before)
    assert (after - ref).abs().max().item() < 1e-5 * ref.abs().max().item()


def test_gradient_checkpointing_same_result_less_memory():
    w, cfg, _ = _pair("vit_small_patch14_dinov2.lvd142m", 14, img=224)
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
    # the forward is the same computation: identical features; the loss kernel adds its CTA partials with atomics
    assert torch.equal(f0, f1) and abs(l0 - l1) < 1e-6 * abs(l0)
    for k in g0:
        assert _cos(g0[k], g1[k]) > 0.9999, k
    assert m1 < 0.6 * m0, (m0, m1)


# ---------------------------------------------------------------------------------------------------------------------
# short run against the oracle loop
# ---------------------------------------------------------------------------------------------------------------------
def test_training_run_matches_oracle():
    """20 AdamW steps (warm-up + cosine schedule): FusedAdamW on the CUDA path against torch.optim.AdamW on the fp32 oracle."""
    from dvt import train_ops
    from dvt.optim import FusedAdamW
    from dvt.utils import misc
    T, B = 20, 2
    w, cfg, sd = _pair("vit_small_patch14_dinov2.lvd142m", 14, depth=3, img=98, seed=8)
    g = torch.Generator().manual_seed(9)
    imgs = torch.randn(4, 3, 98, 98, generator=g)
    targets = torch.randn(4, 7, 7, cfg.embed_dim, generator=g)
    batches = [torch.randint(0, 4, (B,), generator=g) for _ in range(T)]
    sched = dict(base_value=1e-3, final_value=1e-5, total_iters=T, warmup_iters=int(T * 0.15), start_warmup_value=0)
    # oracle
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
    # CUDA path
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
# command line
# ---------------------------------------------------------------------------------------------------------------------
def test_stage3_cli_trains_and_checkpoints(tmp_path, capsys, monkeypatch):
    """main_distillation.py on an ImageFolder of 8 synthetic 70 x 70 PNGs (one mirror-symmetric image, so that every batch,
    flipped or not, is the same and the loss trajectory is not sampling noise), the student and the teacher's backbone loaded
    from the same saved ViT-S/14 (LayerScale 1), a teacher denoiser in the stage-2 checkpoint layout: the loss falls, the
    checkpoints have the reference's layout and load strictly into a fresh wrapper, `--resume` continues."""
    from PIL import Image
    import dvt.models as DVT
    from dvt.models import vit_wrapper as VW
    sys.path.insert(0, ROOT)
    import main_distillation as M
    ident = "vit_small_patch14_dinov2.lvd142m"
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
    den = DVT.Denoiser(5, 5, 384, vit=None, num_blocks=1)
    torch.save({"denoiser": den.state_dict(), "optimizer": {}, "step": 0}, tmp_path / "denoiser.pth")
    argv = ["--model", ident, "--denoiser_ckpt", str(tmp_path / "denoiser.pth"), "--input_size", "70", "--stride_size", "14",
            "--data_root", str(tmp_path / "data"), "--batch_size", "4", "--num_iterations", "20", "--blr", "0.002",
            "--output_root", str(tmp_path / "work"), "--run_name", "t", "--save_freq", "10", "--num_workers", "0",
            "--log_freq", "5"]
    M.main(M.get_args(argv))
    out = capsys.readouterr().out
    vals = [float(ln.split("loss: ")[1].split()[0]) for ln in out.splitlines() if ln.startswith("Train [")]
    assert len(vals) >= 4 and vals[-1] < vals[0], vals
    ck_dir = tmp_path / "work" / "denosing-vit" / "t" / "checkpoints"
    assert sorted(os.listdir(ck_dir)) == ["ckpt_000000.pth", "ckpt_000010.pth", "ckpt_000019.pth", "latest.pth"]
    assert os.path.islink(ck_dir / "latest.pth")
    ck = torch.load(str(ck_dir / "latest.pth"), map_location="cpu")
    assert set(ck) == {"model", "optimizer", "step"} and ck["step"] == 19
    assert all(k.startswith("model.") for k in ck["model"]) and "model.blocks.0.ls1.gamma" in ck["model"]
    fresh = DVT.PretrainedViTWrapper(ident, stride=14, allow_random_init=True)
    fresh.load_state_dict(ck["model"], strict=True)
    assert set(ck["optimizer"]) == {"state", "param_groups"}
    i = argv.index("--num_iterations")
    M.main(M.get_args(argv[:i + 1] + ["24"] + argv[i + 2:] + ["--resume", str(ck_dir / "latest.pth")]))
    out2 = capsys.readouterr().out
    assert "Resumed from" in out2 and "at step 20" in out2 and os.path.isfile(ck_dir / "ckpt_000023.pth")
