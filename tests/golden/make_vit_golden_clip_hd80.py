"""Generates tests/golden/vit_hf_clip.npz and tests/golden/vit_hf_hd80.npz: outputs of INDEPENDENT implementations of
the two ViT variants added for the CLIP towers and ViT-H/14 MAE (random-init, no checkpoint), used to pin the pre_norm /
bias-less patch embedding / eps 1e-5 path and the head_dim-80 path of the oracle extension in tests/vit_oracle_ext.py.

  vit_hf_clip.npz  transformers.CLIPVisionModel, hidden_act="gelu" (erf GELU, what timm 1.0.7's vit_base_patch16_clip_*
                   definitions run), layer_norm_eps=1e-5.  pre_layrnorm -> norm_pre, q/k/v_proj -> attn.qkv,
                   class_embedding -> cls_token [1, 1, C], no patch bias.  HF applies post_layernorm to the pooled token
                   only, so the norm=True target is post_layernorm(last_hidden_state).
  vit_hf_hd80.npz  transformers.ViTModel(add_pooling_layer=False), hidden_size 160 with 2 heads (head_dim 80),
                   layer_norm_eps=1e-6 (HF's default is 1e-12).  last_hidden_state has the final LayerNorm applied.

Both store the input, the timm-named fp32 weights, the norm=True target (`hf_last_hidden_state`, all tokens), the output
of block 0 without the final norm (`hf_block0`) and the transformers version.  Native grid only: HF's position
interpolation is not timm's antialiased resample.

Run on CPU:  python tests/golden/make_vit_golden_clip_hd80.py
"""
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))


def _perturb(model, g):
    """Non-trivial values everywhere (HF init leaves biases at 0 and LayerNorms at 1 / 0).  Every weight is then rounded
    to a bf16-representable fp32 value: the fixture compresses to half its size, and nothing else changes."""
    with torch.no_grad():
        for n, p in model.named_parameters():
            if ("norm" in n or "layrnorm" in n) and n.endswith("weight"):
                p.copy_(1.0 + 0.1 * torch.randn(p.shape, generator=g))
            elif (n.endswith("bias") or "embedding" in n or "token" in n) and not ("patch" in n and n.endswith("weight")):
                p.copy_(torch.randn(p.shape, generator=g) * 0.05)
            p.copy_(p.bfloat16().float())


def _save(name, x, target, block0, sd, meta):
    import transformers
    arrays = {"x": x.numpy(), "hf_last_hidden_state": target.numpy(), "hf_block0": block0.numpy(),
              "meta": np.array(meta, dtype=np.int64), "transformers_version": np.array(transformers.__version__)}
    for k, v in sd.items():
        arrays["w:" + k] = v.detach().float().contiguous().numpy()
    path = os.path.join(HERE, f"vit_hf_{name}.npz")
    np.savez_compressed(path, **arrays)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB", "transformers", transformers.__version__)


def make_clip(seed=0):
    import transformers
    torch.manual_seed(seed)
    C, depth, heads, hid, img, P = 64, 2, 1, 256, 64, 16
    cfg = transformers.CLIPVisionConfig(hidden_size=C, intermediate_size=hid, num_hidden_layers=depth,
                                        num_attention_heads=heads, image_size=img, patch_size=P, hidden_act="gelu",
                                        layer_norm_eps=1e-5, attention_dropout=0.0)
    model = transformers.CLIPVisionModel(cfg).eval()
    _perturb(model, torch.Generator().manual_seed(seed + 1))
    x = torch.randn(2, 3, img, img, generator=torch.Generator().manual_seed(seed + 2))
    vm = model.vision_model
    with torch.no_grad():
        out = model(pixel_values=x, output_hidden_states=True)
        target = vm.post_layernorm(out.last_hidden_state)
        block0 = out.hidden_states[1]          # hidden_states[0] is the encoder input (after pre_layrnorm)
    hf = {k: v for k, v in vm.state_dict().items()}
    sd = {
        "cls_token": hf["embeddings.class_embedding"].reshape(1, 1, C),
        "pos_embed": hf["embeddings.position_embedding.weight"].unsqueeze(0),
        "patch_embed.proj.weight": hf["embeddings.patch_embedding.weight"],
        "norm_pre.weight": hf["pre_layrnorm.weight"],
        "norm_pre.bias": hf["pre_layrnorm.bias"],
        "norm.weight": hf["post_layernorm.weight"],
        "norm.bias": hf["post_layernorm.bias"],
    }
    assert "embeddings.patch_embedding.bias" not in hf
    for i in range(depth):
        h, t = f"encoder.layers.{i}.", f"blocks.{i}."
        a = h + "self_attn."
        sd[t + "attn.qkv.weight"] = torch.cat([hf[a + "q_proj.weight"], hf[a + "k_proj.weight"], hf[a + "v_proj.weight"]])
        sd[t + "attn.qkv.bias"] = torch.cat([hf[a + "q_proj.bias"], hf[a + "k_proj.bias"], hf[a + "v_proj.bias"]])
        sd[t + "attn.proj.weight"] = hf[a + "out_proj.weight"]
        sd[t + "attn.proj.bias"] = hf[a + "out_proj.bias"]
        sd[t + "norm1.weight"], sd[t + "norm1.bias"] = hf[h + "layer_norm1.weight"], hf[h + "layer_norm1.bias"]
        sd[t + "norm2.weight"], sd[t + "norm2.bias"] = hf[h + "layer_norm2.weight"], hf[h + "layer_norm2.bias"]
        sd[t + "mlp.fc1.weight"], sd[t + "mlp.fc1.bias"] = hf[h + "mlp.fc1.weight"], hf[h + "mlp.fc1.bias"]
        sd[t + "mlp.fc2.weight"], sd[t + "mlp.fc2.bias"] = hf[h + "mlp.fc2.weight"], hf[h + "mlp.fc2.bias"]
    _save("clip", x, target, block0, sd, [C, depth, heads, P, img, hid, 0, 0])


def make_hd80(seed=0):
    import transformers
    torch.manual_seed(seed)
    C, depth, heads, hid, img, P = 160, 2, 2, 160, 56, 14
    cfg = transformers.ViTConfig(hidden_size=C, num_hidden_layers=depth, num_attention_heads=heads, intermediate_size=hid,
                                 image_size=img, patch_size=P, hidden_act="gelu", layer_norm_eps=1e-6, qkv_bias=True,
                                 hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    model = transformers.ViTModel(cfg, add_pooling_layer=False).eval()
    _perturb(model, torch.Generator().manual_seed(seed + 1))
    x = torch.randn(2, 3, img, img, generator=torch.Generator().manual_seed(seed + 2))
    with torch.no_grad():
        out = model(pixel_values=x, output_hidden_states=True)
        target = out.last_hidden_state         # final LayerNorm applied
        block0 = out.hidden_states[1]
    hf = {k: v for k, v in model.state_dict().items()}
    sd = {
        "cls_token": hf["embeddings.cls_token"],
        "pos_embed": hf["embeddings.position_embeddings"],
        "patch_embed.proj.weight": hf["embeddings.patch_embeddings.projection.weight"],
        "patch_embed.proj.bias": hf["embeddings.patch_embeddings.projection.bias"],
        "norm.weight": hf["layernorm.weight"],
        "norm.bias": hf["layernorm.bias"],
    }
    for i in range(depth):
        h, t = f"encoder.layer.{i}.", f"blocks.{i}."
        a = h + "attention.attention."
        sd[t + "attn.qkv.weight"] = torch.cat([hf[a + "query.weight"], hf[a + "key.weight"], hf[a + "value.weight"]])
        sd[t + "attn.qkv.bias"] = torch.cat([hf[a + "query.bias"], hf[a + "key.bias"], hf[a + "value.bias"]])
        sd[t + "attn.proj.weight"] = hf[h + "attention.output.dense.weight"]
        sd[t + "attn.proj.bias"] = hf[h + "attention.output.dense.bias"]
        sd[t + "norm1.weight"], sd[t + "norm1.bias"] = hf[h + "layernorm_before.weight"], hf[h + "layernorm_before.bias"]
        sd[t + "norm2.weight"], sd[t + "norm2.bias"] = hf[h + "layernorm_after.weight"], hf[h + "layernorm_after.bias"]
        sd[t + "mlp.fc1.weight"], sd[t + "mlp.fc1.bias"] = hf[h + "intermediate.dense.weight"], hf[h + "intermediate.dense.bias"]
        sd[t + "mlp.fc2.weight"], sd[t + "mlp.fc2.bias"] = hf[h + "output.dense.weight"], hf[h + "output.dense.bias"]
    _save("hd80", x, target, block0, sd, [C, depth, heads, P, img, hid, 0, 0])


if __name__ == "__main__":
    make_clip()
    make_hd80()
