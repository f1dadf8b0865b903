"""The DINOv3 backbones on the GPU: the QKV GEMM with the 2-D RoPE epilogue and its backward against float64, the
wrapper's inference forward against transformers.DINOv3ViTModel (golden vit_hf_dinov3.npz) and against the RoPE oracle
(tests/vit_oracle_rope.py) at stride < patch, stage-3 gradients of every parameter against autograd through the oracle, a
short training run, deterministic training, and every CLI end to end with a randomly initialised backbone.
Tolerances as tests/test_distill_gpu.py: bf16 tensor-core GEMMs with fp32 accumulation against fp32 / fp64 references."""
import contextlib
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import vit_oracle_rope as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
SMALL = "vit_small_patch16_dinov3.lvd1689m"


def _dev_ok():
    from dvt import _lib
    torch.cuda.synchronize()
    assert _lib.device_error() == 0


@contextlib.contextmanager
def _impl(impl):
    from dvt import _lib
    _lib.check(_lib.lib().dvt_set_debug_impl(impl), "dvt_set_debug_impl")
    try:
        yield
    finally:
        _lib.lib().dvt_set_debug_impl(-1)


def _cos(a, b):
    return F.cosine_similarity(a.flatten().double(), b.flatten().double(), dim=0).item()


def _min_cos(a, b):
    C = a.shape[-1]
    return F.cosine_similarity(a.reshape(-1, C).double().cpu(), b.reshape(-1, C).double().cpu(), dim=-1).min().item()


# ---------------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------------
def _rotate64(t, rope, B, ntok, prefix, C, transpose=False):
    """float64 restatement of the rotation on the q / k columns of t [B * ntok, 3C] (transpose: R^T)."""
    t = t.double().clone().view(B, ntok, 3 * C)
    cs = rope.double()
    c, s = cs[:, :32], cs[:, 32:]
    if transpose:
        s = -s
    for h in range(2 * C // 64):
        lo = t[:, prefix:, 64 * h:64 * h + 32].clone()
        hi = t[:, prefix:, 64 * h + 32:64 * h + 64].clone()
        t[:, prefix:, 64 * h:64 * h + 32] = lo * c - hi * s
        t[:, prefix:, 64 * h + 32:64 * h + 64] = hi * c + lo * s
    return t.view(B * ntok, 3 * C)


CASES = [  # (B, h, w, prefix, C): ragged M, tiles spanning image boundaries with prefix rows inside, batch > 1
    (3, 5, 7, 5, 128),
    (2, 14, 14, 5, 384),
    (1, 4, 4, 1, 768),
    (5, 3, 9, 0, 256),
]


@pytest.mark.parametrize("impl", [0, 1], ids=["tc", "simt"])
@pytest.mark.parametrize("B,h,w,prefix,C", CASES)
def test_qkv_rope_epilogue_matches_float64(impl, B, h, w, prefix, C):
    from dvt import train_ops
    from dvt.models import vit_wrapper as VW
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + C + prefix)
    ntok = prefix + h * w
    M = B * ntok
    x = torch.randn(M, C, device="cuda", generator=g).bfloat16()
    wq = (torch.randn(3 * C, C, device="cuda", generator=g) / C ** 0.5).bfloat16()
    bias = torch.randn(3 * C, device="cuda", generator=g)
    rope = VW.rope_table(h, w).cuda()
    with _impl(impl):
        got = train_ops.gemm_qkv_rope(x, wq, bias, rope, B, prefix, C // 64)
    _dev_ok()
    ref = _rotate64(x.double() @ wq.double().t() + bias.double(), rope, B, ntok, prefix, C)
    err = (got.double() - ref).abs()
    assert err.max().item() <= 1e-2 * ref.abs().max().item()
    assert (err <= 2 ** -7 * ref.abs() + 1e-3 * ref.abs().max()).all(), err.max()
    # the v columns and the prefix rows are the plain projection
    plain = (x.double() @ wq.double().t() + bias.double()).view(B, ntok, 3 * C)
    gv = got.double().view(B, ntok, 3 * C)
    assert ((gv[:, :, 2 * C:] - plain[:, :, 2 * C:]).abs() <= 2 ** -7 * plain[:, :, 2 * C:].abs() + 1e-3).all()
    if prefix:
        assert ((gv[:, :prefix] - plain[:, :prefix]).abs() <= 2 ** -7 * plain[:, :prefix].abs() + 1e-3).all()


@pytest.mark.parametrize("B,h,w,prefix,C", CASES)
def test_rope_backward_is_the_transpose(B, h, w, prefix, C):
    from dvt import train_ops
    from dvt.models import vit_wrapper as VW
    g = torch.Generator(device="cuda").manual_seed(7 + B + C)
    ntok = prefix + h * w
    M = B * ntok
    y = torch.randn(M, 3 * C, device="cuda", generator=g).bfloat16()
    x = torch.randn(M, 3 * C, device="cuda", generator=g).double()
    rope = VW.rope_table(h, w).cuda()
    z = train_ops.rope_bwd_(y.clone(), rope, B, prefix, C // 64)
    z2 = train_ops.rope_bwd_(y.clone(), rope, B, prefix, C // 64)
    _dev_ok()
    assert torch.equal(z, z2)
    ref = _rotate64(y, rope, B, ntok, prefix, C, transpose=True)
    # R^T y to the one bf16 rounding of the output (the rotation itself in fp32)
    assert ((z.double() - ref).abs() <= 2 ** -8 * ref.abs() + 1e-6).all()
    zv, yv = z.view(B, ntok, 3 * C), y.view(B, ntok, 3 * C)
    assert torch.equal(zv[:, :, 2 * C:], yv[:, :, 2 * C:]) and torch.equal(zv[:, :prefix], yv[:, :prefix])
    # <R x, y> = <x, R^T y>
    lhs = (_rotate64(x, rope, B, ntok, prefix, C) * y.double()).sum().item()
    rhs = (x * ref).sum().item()
    assert abs(lhs - rhs) <= 1e-9 * (x.abs() * y.double().abs()).sum().item()
    got = (x * z.double()).sum().item()
    assert abs(got - rhs) <= 2 ** -8 * (x.abs() * ref.abs()).sum().item()


# ---------------------------------------------------------------------------------------------------------------------
# inference forward
# ---------------------------------------------------------------------------------------------------------------------
def _golden_model():
    from dvt.models import vit_wrapper as VW
    z, hf, xs = R.load_golden(os.path.join(GOLD, "vit_hf_dinov3.npz"))
    C, depth, heads, patch, hidden, reg = [int(v) for v in z["meta"]]
    a = dict(VW.DINOV3_ARCHS[SMALL])
    a.update(embed=C, depth=depth, heads=heads, mlp=hidden, img=64)
    model = VW.B200VisionTransformer(SMALL, patch, a)
    model.load_state_dict(hf, strict=True)
    cfg = R.RopeViTConfig(C, depth, heads, patch, 64, hidden, num_reg_tokens=reg, no_embed_class=True, ln_eps=1e-5)
    return (z, xs), model.cuda(), cfg, {k: v.detach().cpu() for k, v in model.state_dict().items()}


@pytest.mark.parametrize("impl", [0, 1], ids=["tc", "simt"])
def test_wrapper_matches_hf_golden(impl):
    (z, xs), model, cfg, _ = _golden_model()
    for i in (0, 1):
        x = xs[i].cuda()
        with _impl(impl):
            feat, prefix = model.forward_intermediates(x, [cfg.depth - 1], return_prefix_tokens=True, norm=True,
                                                       output_fmt="NLC", intermediates_only=True)[0]
            f0, p0 = model.forward_intermediates(x, [0], return_prefix_tokens=True, norm=False, output_fmt="NLC",
                                                 intermediates_only=True)[0]
            f1 = model.forward_intermediates(x, [cfg.depth - 1], norm=False, output_fmt="NCHW", intermediates_only=True)[0]
        _dev_ok()
        H, W = x.shape[2:]
        assert f1.shape == (2, cfg.embed_dim, H // 16, W // 16)
        for got, ref in ((torch.cat([prefix, feat], 1), z[f"last{i}"]), (torch.cat([p0, f0], 1), z[f"hidden{i}"][1]),
                         (f1.permute(0, 2, 3, 1).reshape(2, -1, cfg.embed_dim), z[f"hidden{i}"][-1][:, 5:])):
            ref = torch.from_numpy(ref).cuda()
            assert got.shape == ref.shape
            assert _min_cos(got, ref) > 0.999, _min_cos(got, ref)
            assert (got - ref).abs().max().item() < 0.05 * ref.abs().max().item()


@pytest.mark.parametrize("stride,hw,B", [(8, (48, 80), 2), (4, (64, 48), 1), (16, (224, 160), 3)])
def test_wrapper_matches_oracle(stride, hw, B):
    """stride < patch (the grid the oracle defines) and a larger image at stride = patch."""
    _, model, cfg, sd = _golden_model()
    model.patch_embed.proj.stride = [stride, stride]
    x = torch.randn(B, 3, *hw, generator=torch.Generator().manual_seed(stride))
    feat, prefix = model.forward_intermediates(x.cuda(), [1], return_prefix_tokens=True, norm=True, output_fmt="NCHW",
                                               intermediates_only=True)[0]
    _dev_ok()
    rf, rp = R.forward_intermediates(sd, cfg, x, [1], stride=stride, return_prefix_tokens=True)[0]
    assert feat.shape == rf.shape
    assert _min_cos(feat.permute(0, 2, 3, 1), rf.permute(0, 2, 3, 1)) > 0.999
    assert _min_cos(prefix, rp) > 0.999


# ---------------------------------------------------------------------------------------------------------------------
# stage 3
# ---------------------------------------------------------------------------------------------------------------------
def _pair(depth=3, seed=0, ident=SMALL, stride=16):
    import dvt.models as DVT
    from dvt.models import vit_wrapper as VW
    a = dict(VW.DINOV3_ARCHS[ident], depth=depth)
    cfg = R.RopeViTConfig(a["embed"], depth, a["heads"], 16, 224, a["mlp"], num_reg_tokens=4, no_embed_class=True,
                          ln_eps=1e-5)
    sd = R.random_state_dict(cfg, seed=seed)
    w = DVT.PretrainedViTWrapper(ident, stride=stride, allow_random_init=True)
    w.model = VW.B200VisionTransformer(ident, 16, a)
    w.model.patch_embed.proj.stride = [stride, stride]
    w.model.load_state_dict(sd, strict=True)
    return w.cuda(), cfg, sd


def _oracle_loss(params, cfg, x, target, stride):
    import vit_oracle_rope as RR
    from oracle import vit as OV
    B = x.shape[0]
    h, w = OV.feat_size(cfg, x.shape[2], x.shape[3], stride)
    t = RR.hidden_states(params, cfg, x, stride)[-1]
    t = F.layer_norm(t, (cfg.embed_dim,), params["norm.weight"], params["norm.bias"], cfg.ln_eps)
    feat = t[:, cfg.num_prefix:].reshape(B, h, w, -1)
    return F.mse_loss(feat, target) + 1 - F.cosine_similarity(feat, target, dim=-1).mean(), feat


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


@pytest.mark.parametrize("stride,hw,ckpt", [(16, (96, 128), False), (8, (64, 80), True)])
def test_vit_gradients_match_oracle(stride, hw, ckpt):
    from oracle import vit as OV
    w, cfg, sd = _pair(depth=3, seed=3, stride=stride)
    w.model.set_grad_checkpointing(ckpt)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 3, *hw, generator=g)
    h, wd = OV.feat_size(cfg, hw[0], hw[1], stride)
    target = torch.randn(2, h, wd, cfg.embed_dim, generator=g)
    params = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    r_loss, r_feat = _oracle_loss(params, cfg, x, target, stride)
    r_loss.backward()
    loss, grads, feat = _our_grads(w, x, target)
    assert _min_cos(feat, r_feat.detach()) > 0.99
    assert abs(loss - r_loss.item()) < 2e-2 * abs(r_loss.item())
    assert set(grads) == set(params)
    C = cfg.embed_dim
    for name, gr in grads.items():
        ref = params[name].grad
        if name.endswith("attn.qkv.bias"):       # no key bias: its gradient slice is zero, the oracle's is not
            assert torch.count_nonzero(gr[C:2 * C]) == 0
            ref = ref.clone()
            ref[C:2 * C] = 0
        c_ = _cos(gr, ref)
        assert c_ > 0.99, f"{name}: gradient cosine {c_}"
        ratio = gr.norm().item() / (ref.norm().item() + 1e-12)
        assert 0.95 < ratio < 1.05, f"{name}: gradient norm ratio {ratio}"


def test_training_forward_equals_inference_forward():
    w, cfg, _ = _pair(depth=2)
    x = torch.randn(2, 3, 80, 112, generator=torch.Generator().manual_seed(1)).cuda()
    ref = w.get_intermediate_layers(x)[0]
    w.set_trainable(True)
    got = w.get_intermediate_layers(x)[0]
    _dev_ok()
    assert got.grad_fn is not None
    assert _min_cos(got.detach().permute(0, 2, 3, 1), ref.permute(0, 2, 3, 1)) > 0.9999


def _train(w, imgs, targets, batches, sched):
    from dvt import train_ops
    from dvt.optim import FusedAdamW
    from dvt.utils import misc
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
    return np.array(logs)


def test_training_run_matches_oracle():
    """30 AdamW steps (warm-up + cosine): FusedAdamW on the CUDA path against torch.optim.AdamW on the fp32 oracle."""
    from dvt.utils import misc
    T, B = 30, 2
    w, cfg, sd = _pair(depth=3, seed=8)
    g = torch.Generator().manual_seed(9)
    imgs = torch.randn(4, 3, 96, 112, generator=g)
    targets = torch.randn(4, 6, 7, cfg.embed_dim, generator=g)
    batches = [torch.randint(0, 4, (B,), generator=g) for _ in range(T)]
    sched = dict(base_value=1e-3, final_value=1e-5, total_iters=T, warmup_iters=int(T * 0.15), start_warmup_value=0)
    params = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    C = cfg.embed_dim
    ropt = torch.optim.AdamW(list(params.values()), betas=(0.9, 0.999), weight_decay=1e-5)
    ref_logs = []
    for s, ids in enumerate(batches):
        for grp in ropt.param_groups:
            grp["lr"] = misc.cosine_schedule(s, **sched)
        loss, _ = _oracle_loss(params, cfg, imgs[ids], targets[ids], 16)
        ropt.zero_grad()
        loss.backward()
        for k, p in params.items():          # DINOv3 has no key bias
            if k.endswith("attn.qkv.bias"):
                p.grad[C:2 * C] = 0
        ropt.step()
        ref_logs.append(loss.item())
    logs = _train(w, imgs, targets, batches, sched)
    ref_logs = np.array(ref_logs)
    assert np.allclose(logs, ref_logs, rtol=0.03, atol=2e-3), np.abs(logs - ref_logs).max()
    assert logs[-1] < logs[0]
    got = {k[len("model."):]: v.detach().cpu() for k, v in w.state_dict().items()}
    for k, v in params.items():
        upd_ref, upd_got = v.detach() - sd[k], got[k] - sd[k]
        if k.endswith("attn.qkv.bias"):
            assert torch.count_nonzero(got[k][C:2 * C]) == 0
            keep = torch.cat([torch.arange(0, C), torch.arange(2 * C, 3 * C)])
            upd_ref, upd_got = upd_ref[keep], upd_got[keep]
        assert _cos(upd_got, upd_ref) > 0.97, f"{k}: update cosine {_cos(upd_got, upd_ref)}"


@pytest.mark.parametrize("ckpt", [False, True], ids=["plain", "checkpointing"])
def test_deterministic_runs_are_bit_identical(ckpt):
    T = 4
    g = torch.Generator().manual_seed(11)
    imgs = torch.randn(4, 3, 64, 96, generator=g)
    targets = torch.randn(4, 4, 6, 384, generator=g)
    batches = [torch.randint(0, 4, (2,), generator=g) for _ in range(T)]
    sched = dict(base_value=1e-3, final_value=1e-5, total_iters=T, warmup_iters=1, start_warmup_value=0)
    runs = []
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(2):
            w, _, _ = _pair(depth=2, seed=12)
            w.model.set_grad_checkpointing(ckpt)
            logs = _train(w, imgs, targets, batches, sched)
            runs.append((logs, {k: v.detach().cpu() for k, v in w.state_dict().items()}))
    finally:
        torch.use_deterministic_algorithms(False)
    (l0, s0), (l1, s1) = runs
    assert np.array_equal(l0, l1)
    for k in s0:
        assert torch.equal(s0[k], s1[k]), k


# ---------------------------------------------------------------------------------------------------------------------
# every stage end to end, randomly initialised backbone
# ---------------------------------------------------------------------------------------------------------------------
def test_denoiser_behind_dinov3_at_stride4():
    import dvt.models as DVT
    vit = DVT.PretrainedViTWrapper(SMALL, stride=4, allow_random_init=True)
    den = DVT.Denoiser(noise_map_height=29, noise_map_width=29, feat_dim=384, vit=vit, num_blocks=1).cuda().eval()
    x = torch.randn(1, 3, 128, 128, generator=torch.Generator().manual_seed(0)).cuda()
    with torch.no_grad():
        raw = vit.get_intermediate_layers(x, n=[11])[0]
        out = den(x)
    _dev_ok()
    assert raw.shape == (1, 384, 29, 29) and torch.isfinite(raw).all()
    assert torch.isfinite(out).all() and out.numel() == 29 * 29 * 384


def test_stage1_2_3_clis(tmp_path, capsys, monkeypatch):
    from PIL import Image
    import dvt.models as DVT
    sys.path.insert(0, ROOT)
    import main_denoiser as MD
    import main_distillation as MS
    import main_img_denoising as MI
    monkeypatch.setenv("DVT_ALLOW_RANDOM_INIT", "1")
    monkeypatch.delenv("DVT_WEIGHTS_DIR", raising=False)
    rs = np.random.RandomState(0)
    data_root = str(tmp_path / "data") + "/"
    rels = ["class0/a.jpg", "class1/b.jpg", "class0/c.jpg", "class1/d.jpg"]
    for rel in rels:
        os.makedirs(os.path.dirname(os.path.join(data_root, rel)), exist_ok=True)
        Image.fromarray(rs.randint(0, 255, (90, 120, 3), dtype=np.uint8)).save(os.path.join(data_root, rel))
    lst = tmp_path / "list.txt"
    lst.write_text("".join(f"{r}\n" for r in rels))
    # stage 1: 80 x 96 at stride 16 -> 5 x 6 maps, C = 384
    argv = ["--model", SMALL, "--input_size", "80", "96", "--stride_size", "16", "--img_path", str(lst), "--data_root",
            data_root, "--save_root", str(tmp_path / "feats"), "--num_views", "4", "--num_iters", "20", "--warmup_iters",
            "2", "--n_levels", "6", "--extract_bsz", "4", "--pixel_bsz", "64", "--output_dir", str(tmp_path / "w1"),
            "--seed", "3", "--collate_out", str(tmp_path / "maps.pt")]
    MI.main(MI.get_args(argv))
    _dev_ok()
    packed = torch.load(str(tmp_path / "maps.pt"))
    assert packed["denoised_feats"].shape == (4, 5, 6, 384) and torch.isfinite(packed["denoised_feats"]).all()
    assert torch.isfinite(packed["raw_feats"]).all()
    capsys.readouterr()
    # stage 2 on the feature store stage 1 wrote (images read with the DINOv3 normalisation), --auto_stride -> 16
    (tmp_path / "list2.txt").write_text("".join(f"{r} 0\n" for r in rels))
    argv = ["--model", SMALL, "--input_size", "80", "96", "--auto_stride", "--data_root", data_root, "--feat_root",
            f"{tmp_path / 'feats'}/denoised_features/{SMALL}/", "--data_list_path", str(tmp_path / "list2.txt"),
            "--batch_size", "2", "--num_iterations", "4", "--output_root", str(tmp_path / "w2"), "--run_name", "d3",
            "--save_freq", "4", "--num_workers", "0", "--log_freq", "1"]
    MD.main(MD.get_args(argv))
    _dev_ok()
    out = capsys.readouterr().out
    vals = [float(ln.split("loss: ")[1].split()[0]) for ln in out.splitlines() if ln.startswith("Train [")]
    assert vals and all(np.isfinite(vals))
    # stage 3 with and without checkpointing / deterministic mode
    den = DVT.Denoiser(4, 4, 384, vit=None, num_blocks=1)
    torch.save({"denoiser": den.state_dict(), "optimizer": {}, "step": 0}, tmp_path / "denoiser.pth")
    for i, extra in enumerate(([], ["--grad_checkpointing", "--deterministic"])):
        argv = ["--model", SMALL, "--denoiser_ckpt", str(tmp_path / "denoiser.pth"), "--input_size", "64", "--stride_size",
                "16", "--data_root", str(tmp_path / "data"), "--batch_size", "2", "--num_iterations", "3", "--blr", "0.001",
                "--output_root", str(tmp_path / "w3"), "--run_name", f"s{i}", "--save_freq", "10", "--num_workers", "0",
                "--log_freq", "1", *extra]
        try:
            MS.main(MS.get_args(argv))
        finally:
            torch.use_deterministic_algorithms(False)
        _dev_ok()
        out = capsys.readouterr().out
        vals = [float(ln.split("loss: ")[1].split()[0]) for ln in out.splitlines() if ln.startswith("Train [")]
        assert len(vals) >= 2 and all(np.isfinite(vals))
        ck = torch.load(str(tmp_path / "w3" / "denosing-vit" / f"s{i}" / "checkpoints" / "latest.pth"), map_location="cpu")
        assert "model.reg_token" in ck["model"] and "model.pos_embed" not in ck["model"]
        assert all(torch.isfinite(v).all() for v in ck["model"].values() if v.is_floating_point())


# the two linear probes: the datasets and command lines of their own tests, with the DINOv3 backbone
@pytest.fixture(scope="module")
def voc(tmp_path_factory):
    import test_dense_eval_gpu as T
    return T.voc.__wrapped__(tmp_path_factory)


@pytest.fixture(scope="module")
def nyu(tmp_path_factory):
    import test_depth_probe_gpu as T
    return T.nyu.__wrapped__(tmp_path_factory)


def _with_backbone(argv):
    i = argv.index("--backbone-type")
    return argv[:i + 1] + [SMALL] + argv[i + 2:]


def test_segmentation_probe_cli(voc, tmp_path, monkeypatch):
    import test_dense_eval_gpu as T
    work = tmp_path / "work"
    T._run(_with_backbone(T._argv(voc, work, 20, ckpt=20)), monkeypatch)
    _dev_ok()
    ck = torch.load(work / "latest.pth", map_location="cpu")
    assert ck["iter"] == 20 and ck["state_dict"]["decode_head.conv_seg.weight"].shape == (4, 384, 1, 1)
    recs, val = T._val_records(work)
    train = [r["loss"] for r in recs if r.get("mode") == "train"]
    assert train and all(np.isfinite(train))
    assert len(val) == 1 and np.isfinite(val[0]["mIoU"]) and len(val[0]["IoU"]) == 4


def test_depth_probe_cli(nyu, tmp_path, monkeypatch):
    import test_depth_probe_gpu as T
    work = tmp_path / "work"
    T._run(_with_backbone(T._argv(nyu, work, 10, ckpt=10, evaluate=10)), monkeypatch)
    _dev_ok()
    ck = torch.load(work / "latest.pth", map_location="cpu")
    assert ck["state_dict"]["decode_head.conv_depth.weight"].shape == (256, 768, 1, 1)   # patch tokens + cls, C = 384
    recs = T._records(work)
    val = [r for r in recs if r.get("mode") == "val"]
    assert len(val) == 1 and all(np.isfinite(val[0][k]) for k in ("a1", "abs_rel", "rmse", "silog"))
    assert all(np.isfinite(r["loss"]) for r in recs if r.get("mode") == "train")
