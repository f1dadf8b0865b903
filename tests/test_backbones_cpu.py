"""The CLIP towers and ViT-H/14 MAE on the CPU: the oracle extension (tests/vit_oracle_ext.py) against independent
implementations (transformers.CLIPVisionModel, transformers.ViTModel at head_dim 80; fixtures written by
tests/golden/make_vit_golden_clip_hd80.py), and the wrapper's construction, key sets and constants."""
import os

import numpy as np
import pytest
import torch

import vit_oracle_ext as E

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CLIP_TAGS = ["vit_base_patch16_clip_384.laion2b_ft_in12k_in1k", "vit_base_patch16_clip_224.openai"]
HUGE = "vit_huge_patch14_224.mae"


def _fixture(name):
    z = np.load(os.path.join(GOLD, f"vit_hf_{name}.npz"))
    e, d, h, p, img, hid, _, _ = [int(v) for v in z["meta"]]
    clip = name == "clip"
    cfg = E.ViTConfig(e, d, h, p, img, hid, layerscale=False, ln_eps=1e-5 if clip else 1e-6, pre_norm=clip,
                      patch_bias=not clip)
    sd = {k[2:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("w:")}
    return z, cfg, sd


@pytest.mark.parametrize("name", ["clip", "hd80"])
def test_oracle_matches_hf(name):
    z, cfg, sd = _fixture(name)
    assert (cfg.embed_dim // cfg.num_heads) == (64 if name == "clip" else 80)
    x = torch.from_numpy(z["x"])
    # norm=True, all tokens (prefix + patches)
    feat, prefix = E.forward_intermediates(sd, cfg, x, [cfg.depth - 1], norm=True, reshape=False, return_prefix_tokens=True)[0]
    ref = torch.from_numpy(z["hf_last_hidden_state"])
    assert (torch.cat([prefix, feat], 1) - ref).abs().max().item() < 1e-5
    # norm=False after block 0
    feat0, prefix0 = E.forward_intermediates(sd, cfg, x, [0], norm=False, reshape=False, return_prefix_tokens=True)[0]
    ref0 = torch.from_numpy(z["hf_block0"])
    assert (torch.cat([prefix0, feat0], 1) - ref0).abs().max().item() < 1e-5
    # reshape=True, patches only
    h, w = E.feat_size(cfg, x.shape[2], x.shape[3], cfg.patch_size)
    m = E.forward_intermediates(sd, cfg, x, [cfg.depth - 1], norm=True)[0]
    assert m.shape == (x.shape[0], cfg.embed_dim, h, w)
    assert (m.flatten(2).transpose(1, 2) - ref[:, 1:]).abs().max().item() < 1e-5


def test_fixture_layout():
    for name in ("clip", "hd80"):
        path = os.path.join(GOLD, f"vit_hf_{name}.npz")
        assert os.path.getsize(path) < 1 << 20
        z = np.load(path)
        assert str(z["transformers_version"])
    _, _, sd = _fixture("clip")
    assert "patch_embed.proj.bias" not in sd and "norm_pre.weight" in sd and sd["cls_token"].shape == (1, 1, 64)


def test_oracle_embed_and_block_stay_differentiable():
    cfg = E.ViTConfig(160, 1, 2, 14, 56, 320, layerscale=False, ln_eps=1e-5, pre_norm=True, patch_bias=False)
    sd = {k: v.requires_grad_(True) for k, v in E.random_state_dict(cfg, seed=3).items()}
    x = torch.randn(1, 3, 56, 56)
    y = E.block(E.embed(sd, cfg, x, 14), sd, 0, cfg).square().sum()
    y.backward()
    assert sd["norm_pre.weight"].grad is not None and sd["patch_embed.proj.weight"].grad is not None
    assert "patch_embed.proj.bias" not in sd


def _wrapper(tag, stride=None):
    import dvt.models as DVT
    return DVT.PretrainedViTWrapper(tag, stride=stride or int(tag.split("patch")[1][:2]), allow_random_init=True)


@pytest.mark.parametrize("tag", CLIP_TAGS + [HUGE])
def test_backbone_constructs_with_timm_keys(tag):
    w = _wrapper(tag)
    cfg = E.CONFIGS[tag]
    keys = set(w.model.state_dict())
    assert keys == set(E.random_state_dict(cfg).keys())
    if tag in CLIP_TAGS:
        assert {"norm_pre.weight", "norm_pre.bias"} <= keys and "patch_embed.proj.bias" not in keys
        assert w.model.patch_embed.proj.bias is None
    else:
        assert not any(k.startswith("norm_pre") for k in keys) and "patch_embed.proj.bias" in keys
        assert len(w.model.blocks) == 32 and w.num_blocks == 32
    # a timm-keyed state dict loads strictly
    w.model.load_state_dict(E.random_state_dict(cfg, seed=1), strict=True)


@pytest.mark.parametrize("tag", CLIP_TAGS + [HUGE])
def test_backbone_constants(tag):
    from dvt.models import vit_wrapper as VW
    w = _wrapper(tag)
    eps = 1e-5 if tag in CLIP_TAGS else 1e-6
    norms = [m for m in w.model.modules() if isinstance(m, torch.nn.LayerNorm)]
    assert norms and all(m.eps == eps for m in norms)
    assert VW.ARCHS[tag]["ln_eps"] == eps
    norm = [t for t in w.transformation.transforms if type(t).__name__ == "Normalize"][0]
    if tag in CLIP_TAGS:
        assert tuple(norm.mean) == (0.48145466, 0.4578275, 0.40821073)
        assert tuple(norm.std) == (0.26862954, 0.26130258, 0.27577711)
    else:
        assert tuple(norm.mean) == (0.485, 0.456, 0.406) and tuple(norm.std) == (0.229, 0.224, 0.225)
    assert w.n_output_dims == (1280 if tag == HUGE else 768)
    assert w.model.embed_dim // VW.ARCHS[tag]["heads"] == (80 if tag == HUGE else 64)
    size = 384 if "384" in tag else 224
    assert w.model.native_grid == (size // w.patch_size,) * 2


def test_existing_archs_keep_their_defaults():
    from dvt.models import vit_wrapper as VW
    for tag, a in VW.ARCHS.items():
        if tag in CLIP_TAGS or tag == HUGE:
            continue
        assert a["pre_norm"] is False and a["patch_bias"] is True and a["ln_eps"] == 1e-6
        assert a["embed"] == 64 * a["heads"]


def test_eva02_still_raises():
    import dvt.models as DVT
    with pytest.raises(NotImplementedError):
        DVT.PretrainedViTWrapper("eva02_base_patch16_clip_224.merged2b", stride=16, allow_random_init=True)


def test_denoiser_cli_accepts_the_new_tags():
    from dvt.models import vit_wrapper as VW
    for tag in CLIP_TAGS + [HUGE]:
        assert tag in VW.MODEL_LIST and tag in VW.ARCHS
