"""The DINOv3 backbones without a GPU: the RoPE oracle (tests/vit_oracle_rope.py) against transformers.DINOv3ViTModel
(fixture tests/golden/make_vit_golden_dinov3.py -> vit_hf_dinov3.npz) in float64, the identifiers, the arch lookup, both
state-dict layouts, the CLIs, and the argument checks of dvt_gemm_qkv_rope / dvt_rope_bwd."""
import json
import os
import sys

import pytest
import torch

import vit_oracle_rope as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
IDS = ["vit_small_patch16_dinov3.lvd1689m", "vit_base_patch16_dinov3.lvd1689m", "vit_large_patch16_dinov3.lvd1689m"]


def _fixture():
    from dvt.models import vit_wrapper as VW
    z, hf, xs = R.load_golden(os.path.join(GOLD, "vit_hf_dinov3.npz"))
    C, depth, heads, patch, hidden, reg = [int(v) for v in z["meta"]]
    cfg = R.RopeViTConfig(C, depth, heads, patch, 64, hidden, num_reg_tokens=reg, no_embed_class=True, ln_eps=1e-5)
    return z, cfg, xs, VW.hf_dinov3_to_container(hf)


@pytest.mark.parametrize("i", [0, 1])
def test_oracle_matches_hf_dinov3(i):
    """Every hidden state and the normed output of both non-square inputs, float64, at the tolerance of the DINOv2 goldens."""
    z, cfg, xs, sd = _fixture()
    sd64 = {k: v.double() for k, v in sd.items()}
    x = xs[i].double()
    hs = R.hidden_states(sd64, cfg, x)
    ref = torch.from_numpy(z[f"hidden{i}"]).double()
    assert len(hs) == ref.shape[0]
    for j, (got, want) in enumerate(zip(hs, ref)):
        assert torch.allclose(got, want, atol=2e-5, rtol=1e-4), (j, (got - want).abs().max())
    feat, prefix = R.forward_intermediates(sd64, cfg, x, [cfg.depth - 1], norm=True, reshape=False,
                                           return_prefix_tokens=True)[0]
    last = torch.from_numpy(z[f"last{i}"]).double()
    assert torch.allclose(torch.cat([prefix, feat], 1), last, atol=2e-5, rtol=1e-4)


def test_fixture_is_non_square_both_ways():
    _, _, xs, _ = _fixture()
    (h0, w0), (h1, w1) = [tuple(x.shape[2:]) for x in xs]
    assert h0 < w0 and h1 > w1


def test_rope_tables_match_hf_and_each_other():
    transformers = pytest.importorskip("transformers")
    from dvt.models import vit_wrapper as VW
    cfg = transformers.DINOv3ViTConfig(hidden_size=128, num_attention_heads=2, patch_size=16, image_size=64)
    emb = transformers.models.dinov3_vit.modeling_dinov3_vit.DINOv3ViTRopePositionEmbedding(cfg).eval()
    for H, W in ((48, 80), (64, 32), (224, 224)):
        cos, sin = emb(torch.zeros(1, 3, H, W))
        oc, os_ = R.rope_cos_sin(H // 16, W // 16)
        assert torch.equal(cos, oc) and torch.equal(sin, os_)
        t = VW.rope_table(H // 16, W // 16)
        assert torch.equal(t[:, :32], oc[:, :32]) and torch.equal(t[:, 32:], os_[:, :32])
        assert torch.equal(oc[:, :32], oc[:, 32:])   # the tiling the kernels rely on: columns d and d + 32 share an angle


def test_stride_below_patch_is_the_denser_grid():
    """stride < patch: the wrapper's grid ((H - P) // s + 1, (W - P) // s + 1) with the same formula (defined here)."""
    cfg = R.RopeViTConfig(128, 1, 2, 16, 64, 256, num_reg_tokens=4, no_embed_class=True, ln_eps=1e-5)
    sd = R.random_state_dict(cfg, seed=1)
    x = torch.randn(1, 3, 48, 80, generator=torch.Generator().manual_seed(0))
    f = R.forward_intermediates(sd, cfg, x, [0], stride=8)[0]
    assert f.shape == (1, 128, 5, 9)
    cos, _ = R.rope_cos_sin(5, 9)
    assert cos.shape == (45, 64)


def test_model_list_keeps_the_reference_list_and_appends_dinov3():
    from dvt.models import vit_wrapper as VW
    with open(os.path.join(GOLD, "api_signatures.json")) as fh:
        ref = json.load(fh)["vit_wrapper.py"]["MODEL_LIST"]
    assert len(ref) == 20 and VW.MODEL_LIST[:20] == ref
    assert VW.MODEL_LIST[20:] == IDS


def test_arch_lookup_knows_both_tables():
    from dvt.models import vit_wrapper as VW
    for tag in IDS:
        assert tag not in VW.ARCHS
        a = VW.arch_of(tag)
        assert a["rope"] and a["reg"] == 4 and a["ls"] and a["ln_eps"] == 1e-5 and a["embed"] == 64 * a["heads"]
        assert a["mlp"] == 4 * a["embed"] and a["mean"] == VW.IMAGENET_MEAN and a["std"] == VW.IMAGENET_STD
    assert [(VW.arch_of(t)["embed"], VW.arch_of(t)["depth"], VW.arch_of(t)["heads"]) for t in IDS] == \
        [(384, 12, 6), (768, 12, 12), (1024, 24, 16)]
    for tag, a in VW.ARCHS.items():
        assert VW.arch_of(tag) is a and not a["rope"]
    with pytest.raises(NotImplementedError):
        VW.arch_of("eva02_base_patch16_clip_224.merged2b")


@pytest.mark.parametrize("tag", IDS)
def test_container_keys_and_width(tag):
    import dvt.models as DVT
    w = DVT.PretrainedViTWrapper(tag, stride=16, allow_random_init=True)
    keys = set(w.model.state_dict())
    assert "pos_embed" not in keys and "cls_token" in keys and "reg_token" in keys
    assert "blocks.0.attn.qkv.weight" in keys and "blocks.0.ls1.gamma" in keys and "norm.weight" in keys
    C = w.model.embed_dim
    assert w.n_output_dims == C and w.model.num_prefix_tokens == 5
    assert torch.count_nonzero(w.model.blocks[0].attn.qkv.bias[C:2 * C]) == 0


def test_hf_and_container_layouts_load_identically(tmp_path, monkeypatch):
    import dvt.models as DVT
    from dvt.models import vit_wrapper as VW
    tag = IDS[0]
    hf = {}
    g = torch.Generator().manual_seed(0)
    ref = DVT.PretrainedViTWrapper(tag, stride=16, allow_random_init=True).model
    C = ref.embed_dim
    # an HF-layout state dict of the same architecture (random values; mask_token must be ignored)
    hf["embeddings.cls_token"] = torch.randn(1, 1, C, generator=g)
    hf["embeddings.mask_token"] = torch.randn(1, 1, C, generator=g)
    hf["embeddings.register_tokens"] = torch.randn(1, 4, C, generator=g)
    hf["embeddings.patch_embeddings.weight"] = torch.randn(C, 3, 16, 16, generator=g)
    hf["embeddings.patch_embeddings.bias"] = torch.randn(C, generator=g)
    for i in range(len(ref.blocks)):
        p = f"model.layer.{i}."
        for n in ("norm1", "norm2"):
            hf[p + n + ".weight"], hf[p + n + ".bias"] = torch.randn(C, generator=g), torch.randn(C, generator=g)
        for n in ("q", "k", "v", "o"):
            hf[p + f"attention.{n}_proj.weight"] = torch.randn(C, C, generator=g)
            if n != "k":
                hf[p + f"attention.{n}_proj.bias"] = torch.randn(C, generator=g)
        hf[p + "layer_scale1.lambda1"], hf[p + "layer_scale2.lambda1"] = torch.rand(C, generator=g), torch.rand(C, generator=g)
        hf[p + "mlp.up_proj.weight"], hf[p + "mlp.up_proj.bias"] = torch.randn(4 * C, C, generator=g), torch.randn(4 * C, generator=g)
        hf[p + "mlp.down_proj.weight"], hf[p + "mlp.down_proj.bias"] = torch.randn(C, 4 * C, generator=g), torch.randn(C, generator=g)
    hf["norm.weight"], hf["norm.bias"] = torch.randn(C, generator=g), torch.randn(C, generator=g)

    a = DVT.PretrainedViTWrapper(tag, stride=16, allow_random_init=True).model
    a.load_state_dict(hf)                                   # HF layout, converted once
    b = DVT.PretrainedViTWrapper(tag, stride=16, allow_random_init=True).model
    b.load_state_dict(VW.hf_dinov3_to_container(hf))         # the container's own layout
    sa, sb = a.state_dict(), b.state_dict()
    assert sa.keys() == sb.keys()
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k
    q = hf["model.layer.0.attention.q_proj.weight"]
    assert torch.equal(sa["blocks.0.attn.qkv.weight"][:C], q)
    assert torch.count_nonzero(sa["blocks.0.attn.qkv.bias"][C:2 * C]) == 0

    # weights from $DVT_WEIGHTS_DIR/<id>.pth, in either layout
    for i, sd in enumerate((hf, sb)):
        d = tmp_path / str(i)
        d.mkdir()
        torch.save(sd, d / f"{tag}.pth")
        monkeypatch.setenv("DVT_WEIGHTS_DIR", str(d))
        w = DVT.PretrainedViTWrapper(tag, stride=16)
        assert w.pretrained_loaded
        for k, v in w.model.state_dict().items():
            assert torch.equal(v, sa[k]), k
    # a stage-3 checkpoint saves the container's own keys (model.<key>)
    ck = {"model." + k: v for k, v in sb.items()}
    d = tmp_path / "ck"
    d.mkdir()
    torch.save(ck, d / f"{tag}.pth")
    monkeypatch.setenv("DVT_WEIGHTS_DIR", str(d))
    assert DVT.PretrainedViTWrapper(tag, stride=16).pretrained_loaded


@pytest.mark.parametrize("tag", IDS)
def test_clis_accept_the_dinov3_ids(tag):
    sys.path.insert(0, ROOT)
    import main_denoiser
    import main_distillation
    import main_img_denoising
    assert main_img_denoising.get_args(["--model", tag, "--stride_size", "16", "--input_size", "512", "--img_path", __file__]).model == tag
    a = main_denoiser.get_args(["--model", tag, "--auto_stride"])
    assert a.model == tag and a.stride_size == 16
    a = main_distillation.get_args(["--denoiser_ckpt", "x.pth", "--model", tag, "--auto_stride"])
    assert a.model == tag and a.stride_size == 16 and a.input_size == [512, 512]


# ---- argument checks (fake pointers, no GPU: a call that passes every check fails with DVT_ERR_CUDA) ----------------
DVT_ERR_INVALID, DVT_ERR_CUDA = 1, 2
BASE = 1 << 32
P = [BASE + i * (1 << 24) for i in range(8)]


def _qkv(L, x=P[0], w=P[1], bias=P[2], rope=P[3], out=P[4], M=2 * 21, C=128, ntok=21, prefix=5, heads=2, head_dim=64,
         ldo=384):
    return L.lib().dvt_gemm_qkv_rope(x, C, w, C, M, C, bias, rope, ntok, prefix, heads, head_dim, out, ldo, None)


def _bwd(L, dqkv=P[0], ld=384, rope=P[1], M=2 * 21, ntok=21, prefix=5, heads=2, head_dim=64):
    return L.lib().dvt_rope_bwd(dqkv, ld, rope, M, ntok, prefix, heads, head_dim, None)


@pytest.fixture(scope="module")
def L():
    if torch.cuda.is_available():
        pytest.skip("fake device pointers: run on a machine without a GPU")
    from dvt import _lib
    return _lib


def _invalid(L, rc, word):
    msg = L.lib().dvt_last_error().decode()
    assert rc == DVT_ERR_INVALID, f"got {rc} ({msg})"
    assert word in msg, msg


@pytest.mark.parametrize("f", [_qkv, _bwd])
def test_rope_calls_valid_reach_the_runtime(L, f):
    assert f(L) == DVT_ERR_CUDA, L.lib().dvt_last_error().decode()
    assert f(L, prefix=0) == DVT_ERR_CUDA


def test_rope_calls_reject_bad_arguments(L):
    _invalid(L, _qkv(L, head_dim=80, C=160), "head_dim")
    _invalid(L, _bwd(L, head_dim=80, ld=480), "head_dim")
    _invalid(L, _qkv(L, prefix=21), "prefix")
    _invalid(L, _bwd(L, prefix=21), "prefix")
    _invalid(L, _qkv(L, prefix=25), "prefix")
    _invalid(L, _qkv(L, rope=P[3] + 4), "RoPE table")
    _invalid(L, _bwd(L, rope=P[1] + 4), "rope")
    _invalid(L, _bwd(L, dqkv=P[0] + 2), "dqkv")
    _invalid(L, _qkv(L, out=P[4] + 2), "out")
    _invalid(L, _qkv(L, bias=P[2] + 4), "bias")
    _invalid(L, _qkv(L, M=43), "multiple")
    _invalid(L, _bwd(L, ld=254), "ld")
    _invalid(L, _qkv(L, rope=None), "null")
