"""The CLIP towers (pre_norm, bias-less patch embedding, eps 1e-5) and ViT-H/14 MAE (head_dim 80) on the GPU: head_dim-80
flash attention forward / backward against torch, the wrapper against the HF fixtures and against the oracle extension
(tests/vit_oracle_ext.py) at real sizes, the denoiser behind them, stage 1, and stage-3 gradients of every parameter.
Tolerances as the existing suites: attention max err < 3e-2 and per-row cosine > 0.9995, ViT per-token cosine > 0.999,
stage-3 gradients cosine >= 0.99 and norm ratio 0.95-1.05."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import vit_oracle_ext as E

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
CLIP224, CLIP384, HUGE = "vit_base_patch16_clip_224.openai", "vit_base_patch16_clip_384.laion2b_ft_in12k_in1k", \
    "vit_huge_patch14_224.mae"


class _impl:
    def __init__(self, impl):
        self.impl = impl

    def __enter__(self):
        from dvt import _lib
        _lib.check(_lib.lib().dvt_set_debug_impl(self.impl))

    def __exit__(self, *a):
        from dvt import _lib
        _lib.check(_lib.lib().dvt_set_debug_impl(-1))


def _dev_ok():
    from dvt import _lib
    torch.cuda.synchronize()
    assert _lib.device_error() == 0


def _min_cos(a, b):
    return F.cosine_similarity(a.float().flatten(0, -2), b.float().flatten(0, -2), dim=-1).min().item()


def _cos(a, b):
    return F.cosine_similarity(a.flatten().double(), b.flatten().double(), dim=0).item()


def _qkv(B, N, heads, D, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(B, N, 3 * heads * D, device="cuda", generator=g) * 1.5).bfloat16()


def _sdpa(qkv, heads, D):
    B, N, _ = qkv.shape
    q, k, v = qkv.float().view(B, N, 3, heads, D).permute(2, 0, 3, 1, 4)
    return F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, N, heads * D), (q, k, v)


# ---------------------------------------------------------------------------------------------------------------------
# attention at head_dim 80
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", [1, 0], ids=["simt", "tc"])
@pytest.mark.parametrize("N,heads,B", [(100, 2, 3), (257, 16, 2), (1370, 2, 1), (5330, 16, 1)])
def test_attention_hd80_forward(impl, N, heads, B):
    from dvt import ops, train_ops
    D = 80
    qkv = _qkv(B, N, heads, D, N + heads)
    ref, (q, k, _) = _sdpa(qkv, heads, D)
    with _impl(impl):
        out = ops.attention(qkv, heads, head_dim=D)
    _dev_ok()
    assert (out.float() - ref).abs().max().item() < 3e-2
    assert _min_cos(out.view(-1, D), ref.view(-1, D)) > 0.9995
    if impl == 0:   # the lse form (training path): same output, lse = log2 sum exp(s * scale)
        out2, lse = train_ops.attention_fwd_lse(qkv, heads, head_dim=D)
        _dev_ok()
        assert torch.equal(out2, out)
        s = (q @ k.transpose(-1, -2)) * D ** -0.5
        ref_lse = torch.logsumexp(s, -1) / np.log(2.0)
        assert (lse - ref_lse).abs().max().item() < 1e-3


def test_attention_hd64_forms_are_the_existing_kernels():
    """head_dim 64: the lse form returns the output of the inference form bit for bit, and always runs the tensor-core
    kernel (same bits under the SIMT debug implementation).  head_dim 72 is rejected."""
    from dvt import _lib, ops, train_ops
    qkv = _qkv(2, 333, 6, 64, 5)
    a = ops.attention(qkv, 6)
    b, lse = train_ops.attention_fwd_lse(qkv, 6)
    with _impl(1):
        c, lse_simt = train_ops.attention_fwd_lse(qkv, 6)
    _dev_ok()
    assert torch.equal(a, b)
    assert torch.equal(b, c) and torch.equal(lse, lse_simt)
    with pytest.raises(_lib.DvtError):
        ops.attention(_qkv(1, 10, 2, 72, 1), 2, head_dim=72)


@pytest.mark.parametrize("N,heads,B", [(100, 2, 3), (257, 16, 2), (1370, 2, 1), (5330, 2, 1)])
def test_attention_hd80_backward(N, heads, B):
    from dvt import train_ops
    D = 80
    qkv = _qkv(B, N, heads, D, 7 * N + heads)
    g = torch.Generator(device="cuda").manual_seed(N)
    dout = torch.randn(B, N, heads * D, device="cuda", generator=g).bfloat16()
    out, lse = train_ops.attention_fwd_lse(qkv, heads, head_dim=D)
    dqkv = train_ops.attention_bwd(qkv, out, dout, lse, heads, head_dim=D)
    again = train_ops.attention_bwd(qkv, out, dout, lse, heads, head_dim=D)
    _dev_ok()
    x = qkv.float().requires_grad_(True)
    ref, _ = _sdpa(x, heads, D)
    ref.backward(dout.float())
    C = heads * D
    for i, name in enumerate(("dq", "dk", "dv")):
        got, want = dqkv[..., i * C:(i + 1) * C].float(), x.grad[..., i * C:(i + 1) * C]
        assert _cos(got, want) >= 0.999, (name, _cos(got, want))
    assert torch.equal(dqkv[..., C:], again[..., C:])        # dK, dV: no atomics, bit-identical repeats


# ---------------------------------------------------------------------------------------------------------------------
# the wrapper against HF and the oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", [1, 0], ids=["simt", "tc"])
@pytest.mark.parametrize("fixture,ident", [("clip", CLIP224), ("hd80", HUGE)])
def test_wrapper_matches_hf_golden(impl, fixture, ident):
    from dvt.models import vit_wrapper as VW
    z = np.load(os.path.join(GOLD, f"vit_hf_{fixture}.npz"))
    e, d, h, p, img, hid, _, _ = [int(v) for v in z["meta"]]
    sd = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w:")}
    arch = dict(VW.ARCHS[ident])
    arch.update(embed=e, depth=d, heads=h, img=img, mlp=hid)
    model = VW.B200VisionTransformer(ident, p, arch)
    model.load_state_dict(sd, strict=True)
    model = model.cuda()
    x = torch.from_numpy(z["x"]).cuda()
    with _impl(impl):
        feat, prefix = model.forward_intermediates(x, [d - 1], return_prefix_tokens=True, norm=True, output_fmt="NLC",
                                                   intermediates_only=True)[0]
        f0, p0 = model.forward_intermediates(x, [0], return_prefix_tokens=True, norm=False, output_fmt="NLC",
                                             intermediates_only=True)[0]
    _dev_ok()
    for got, ref in ((torch.cat([prefix, feat], 1), z["hf_last_hidden_state"]), (torch.cat([p0, f0], 1), z["hf_block0"])):
        ref = torch.from_numpy(ref).cuda()
        assert got.shape == ref.shape
        assert _min_cos(got, ref) > 0.999, _min_cos(got, ref)
        assert (got - ref).abs().max().item() < 0.1


def _wrapper_from_sd(ident, sd, stride):
    import dvt.models as DVT
    w = DVT.PretrainedViTWrapper(ident, stride=stride, allow_random_init=True)
    w.model.load_state_dict(sd, strict=True)
    return w.cuda().eval()


@pytest.mark.parametrize("impl", [1, 0], ids=["simt", "tc"])
@pytest.mark.parametrize("ident,size,stride,B", [
    (CLIP384, 384, 16, 1),          # native grid
    (CLIP224, 224, 8, 2),           # overlapping patches: resampled position grid 14 -> 27
    (HUGE, 224, 14, 2),             # native grid, head_dim 80
    (HUGE, 224, 7, 1),              # stride 7: 31 x 31 patches
])
def test_wrapper_matches_oracle(impl, ident, size, stride, B):
    cfg = E.CONFIGS[ident]
    sd = E.random_state_dict(cfg, seed=1)
    x = torch.randn(B, 3, size, size, generator=torch.Generator().manual_seed(2))
    layer, mid_layer = cfg.depth - 1, cfg.depth // 2
    ref, ref_mid = E.forward_intermediates(sd, cfg, x, [mid_layer, layer], stride=stride)[::-1]
    ref_mid_raw = E.forward_intermediates(sd, cfg, x, [mid_layer], stride=stride, norm=False)[0]
    w = _wrapper_from_sd(ident, sd, stride)
    with _impl(impl):
        got = w.get_intermediate_layers(x.cuda(), n=[layer], reshape=True)[-1]
        mid = w.get_intermediate_layers(x.cuda(), n=[mid_layer], reshape=True)[-1]
        mid_raw = w.get_intermediate_layers(x.cuda(), n=[mid_layer], reshape=True, norm=False)[-1]
    _dev_ok()
    for g_, r_ in ((got, ref), (mid, ref_mid), (mid_raw, ref_mid_raw)):
        assert g_.shape == r_.shape
        c = _min_cos(g_.permute(0, 2, 3, 1).cpu(), r_.permute(0, 2, 3, 1))
        assert c > 0.999, c


@pytest.mark.parametrize("ident,size,stride", [(CLIP224, 224, 16), (HUGE, 224, 14)])
def test_denoiser_behind_the_new_backbones(ident, size, stride):
    import dvt.models as DVT
    from oracle import denoiser as OD
    cfg = E.CONFIGS[ident]
    vsd = E.random_state_dict(cfg, seed=5)
    vit = DVT.PretrainedViTWrapper(ident, stride=stride, allow_random_init=True)
    vit.model.load_state_dict(vsd, strict=True)
    C = vit.n_output_dims
    h, w = E.feat_size(cfg, size, size, stride)
    sd = OD.random_state_dict(C, (h, w), 1, seed=9)
    m = DVT.Denoiser(h, w, C, vit=vit, enable_pe=True)
    m.load_state_dict({**sd, **{"vit." + k: v for k, v in vit.state_dict().items()}}, strict=True)
    m = m.cuda().eval()
    x = torch.randn(1, 3, size, size, generator=torch.Generator().manual_seed(4))
    with torch.no_grad():
        got, cls = m(x.cuda(), return_class_token=True)
    _dev_ok()
    feats, prefix = E.forward_intermediates(vsd, cfg, x, [cfg.depth - 1], stride=stride, return_prefix_tokens=True)[0]
    ref = OD.forward(sd, feats.permute(0, 2, 3, 1), (h, w))
    assert got.shape == (1, h, w, C)
    assert _min_cos(got.cpu(), ref) > 0.999
    assert _min_cos(cls.cpu()[:, None], prefix[:, :1]) > 0.999


def test_stage1_pipeline_with_clip():
    """One image through Stage1Pipeline with a short fit on the CLIP tower: the raw maps are the backbone's features."""
    import dvt.models as DVT
    from dvt.stage1 import Stage1Config, Stage1Pipeline
    torch.manual_seed(0)
    vit = DVT.PretrainedViTWrapper(CLIP224, stride=16, allow_random_init=True)
    vit.model.load_state_dict(E.random_state_dict(E.CONFIGS[CLIP224], seed=2), strict=True)
    vit = vit.cuda().eval()
    cfg = Stage1Config(num_iters=40, warmup_iters=4, n_levels=6, extract_bsz=4, pixel_bsz=64, graph_steps=5)
    pipe = Stage1Pipeline(vit, layer_index=11, input_size=(64, 80), cfg=cfg)
    g = torch.Generator(device="cuda").manual_seed(3)
    V = 4
    views = torch.randn(V, 3, 64, 80, device="cuda", generator=g)
    coords = torch.rand(V, pipe.h, pipe.w, 2, device="cuda", generator=g)
    n_rows = V * pipe.h * pipe.w
    res = pipe.run_images(1, lambda i: views, lambda i: coords,
                          lambda i: np.random.RandomState(i).randint(0, n_rows, (cfg.num_iters, cfg.pixel_bsz)),
                          lambda i, out: (out["denoised_feats"].cpu(), out["raw"].cpu()))
    _dev_ok()
    den, raw = res[0]
    assert torch.isfinite(den).all() and torch.isfinite(raw).all()
    direct = vit.get_intermediate_layers(views, n=[11], reshape=True)[-1].permute(0, 2, 3, 1).cpu()
    assert raw.shape == direct[-1].shape and raw.shape[-1] == 768          # raw: the last view's feature map
    assert _min_cos(raw.reshape(-1, 768), direct[-1].reshape(-1, 768)) > 0.999


# ---------------------------------------------------------------------------------------------------------------------
# stage 3: every parameter gradient against autograd through the fp32 oracle extension
# ---------------------------------------------------------------------------------------------------------------------
GRAD_CASES = {
    "clip-b16-depth3": dict(ident=CLIP224, depth=3, img=None, stride=16, hw=(96, 112)),
    "clip-b16-depth2-stride8": dict(ident=CLIP384, depth=2, img=None, stride=8, hw=(64, 64)),
    "hd80-depth2": dict(ident=HUGE, depth=2, img=None, stride=14, hw=(98, 112)),
}


def _grad_pair(ident, depth, stride, seed):
    import dvt.models as DVT
    from dvt.models import vit_wrapper as VW
    a = dict(VW.ARCHS[ident])
    a["depth"] = depth
    base = E.CONFIGS[ident]
    cfg = E.ViTConfig(base.embed_dim, depth, base.num_heads, base.patch_size, base.native_img, base.mlp_hidden,
                      layerscale=False, ln_eps=base.ln_eps, pre_norm=base.pre_norm, patch_bias=base.patch_bias)
    sd = E.random_state_dict(cfg, seed=seed)
    w = DVT.PretrainedViTWrapper(ident, stride=stride, allow_random_init=True)
    w.model = VW.B200VisionTransformer(ident, base.patch_size, a)
    w.model.patch_embed.proj.stride = [stride, stride]
    w.model.load_state_dict(sd, strict=True)
    return w.cuda(), cfg, sd


def _oracle_grads(sd, cfg, x, target, stride):
    params = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    B, _, H, W = x.shape
    h, w = E.feat_size(cfg, H, W, stride)
    t = E.embed(params, cfg, x, stride)
    for i in range(cfg.depth):
        t = E.block(t, params, i, cfg)
    t = F.layer_norm(t, (cfg.embed_dim,), params["norm.weight"], params["norm.bias"], cfg.ln_eps)
    feat = t[:, cfg.num_prefix:].reshape(B, h, w, -1)
    loss = F.mse_loss(feat, target) + 1 - F.cosine_similarity(feat, target, dim=-1).mean()
    loss.backward()
    return loss.item(), {k: p.grad for k, p in params.items()}, feat.detach()


@pytest.mark.parametrize("checkpoint", [False, True], ids=["plain", "ckpt"])
@pytest.mark.parametrize("case", list(GRAD_CASES))
def test_vit_gradients_match_oracle(case, checkpoint):
    from dvt import train_ops
    c = GRAD_CASES[case]
    w, cfg, sd = _grad_pair(c["ident"], c["depth"], c["stride"], seed=3)
    g = torch.Generator().manual_seed(4)
    x = torch.randn(2, 3, *c["hw"], generator=g)
    h, wd = E.feat_size(cfg, c["hw"][0], c["hw"][1], c["stride"])
    target = torch.randn(2, h, wd, cfg.embed_dim, generator=g)
    r_loss, r_grads, r_feat = _oracle_grads(sd, cfg, x, target, c["stride"])
    w.set_trainable(True)
    w.model.set_grad_checkpointing(checkpoint)
    pred = w.get_intermediate_layers(x.cuda())[0].permute(0, 2, 3, 1)
    loss, _, _ = train_ops.denoise_loss(pred, target.cuda())
    loss.backward()
    _dev_ok()
    grads = {k[len("model."):]: p.grad.detach().cpu() for k, p in w.named_parameters()}
    assert _min_cos(pred.detach().cpu().reshape(-1, cfg.embed_dim), r_feat.reshape(-1, cfg.embed_dim)) > 0.99
    assert abs(loss.item() - r_loss) < 2e-2 * abs(r_loss)
    assert set(grads) == set(r_grads)
    if cfg.pre_norm:
        assert "norm_pre.weight" in grads and "patch_embed.proj.bias" not in grads
    for name, gr in grads.items():
        c_ = _cos(gr, r_grads[name])
        assert c_ > 0.99, f"{name}: gradient cosine {c_}"
        ratio = gr.norm().item() / (r_grads[name].norm().item() + 1e-12)
        assert 0.95 < ratio < 1.05, f"{name}: gradient norm ratio {ratio}"


def test_distillation_cli_with_clip(tmp_path, capsys, monkeypatch):
    """main_distillation.py runs a few steps end to end on a CLIP tag with a randomly initialised backbone."""
    from PIL import Image
    import dvt.models as DVT
    sys.path.insert(0, ROOT)
    import main_distillation as M
    monkeypatch.setenv("DVT_ALLOW_RANDOM_INIT", "1")
    monkeypatch.delenv("DVT_WEIGHTS_DIR", raising=False)
    rs = np.random.RandomState(0)
    for i in range(4):
        d = tmp_path / "data" / f"class{i % 2}"
        d.mkdir(parents=True, exist_ok=True)
        Image.fromarray(rs.randint(0, 255, (64, 64, 3), dtype=np.uint8)).save(d / f"{i}.png")
    den = DVT.Denoiser(4, 4, 768, vit=None, num_blocks=1)
    torch.save({"denoiser": den.state_dict(), "optimizer": {}, "step": 0}, tmp_path / "denoiser.pth")
    argv = ["--model", CLIP224, "--denoiser_ckpt", str(tmp_path / "denoiser.pth"), "--input_size", "64", "--stride_size",
            "16", "--data_root", str(tmp_path / "data"), "--batch_size", "2", "--num_iterations", "4", "--blr", "0.001",
            "--output_root", str(tmp_path / "work"), "--run_name", "clip", "--save_freq", "10", "--num_workers", "0",
            "--log_freq", "1"]
    M.main(M.get_args(argv))
    _dev_ok()
    out = capsys.readouterr().out
    vals = [float(ln.split("loss: ")[1].split()[0]) for ln in out.splitlines() if ln.startswith("Train [")]
    assert len(vals) >= 2 and all(np.isfinite(vals))
    ck = torch.load(str(tmp_path / "work" / "denosing-vit" / "clip" / "checkpoints" / "latest.pth"), map_location="cpu")
    assert "model.norm_pre.weight" in ck["model"] and "model.patch_embed.proj.bias" not in ck["model"]
