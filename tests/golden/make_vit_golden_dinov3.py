"""Generates tests/golden/vit_hf_dinov3.npz: outputs of an INDEPENDENT implementation of the DINOv3 ViT
(`transformers.DINOv3ViTModel`, random-init, no checkpoint, eval mode) used to pin the 2-D RoPE of
tests/vit_oracle_rope.py and the DINOv3 backbone of the wrapper.

Run in the build container:  python tests/golden/make_vit_golden_dinov3.py
The .npz holds HF's own state dict (key layout of `DINOv3ViTModel.state_dict()`), two non-square inputs (48x80 and
64x32: a swapped h / w changes the result), every hidden state of each (`output_hidden_states=True`: the token assembly,
then the output of each layer) and the normed `last_hidden_state` (float32).  Tiny sizes (width 128, 2 heads of 64,
depth 2, 4 registers, patch 16, MLP 256), and values chosen so that they are stored exactly in few bytes, keep the
fixture small: every parameter is set to int8 * 2^e before the run (per tensor, e the smallest power of two that fits
its range; stored as "hf:<key>" int8 and "scale:<key>" float32), the inputs are rounded to float16 before the run and
stored as float16.  tests/vit_oracle_rope.py `load_golden` reads it back to the float32 values the model ran with.
"""
import math
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
SIZES = ((48, 80), (64, 32))


def make(seed=0):
    import transformers
    torch.manual_seed(seed)
    cfg = transformers.DINOv3ViTConfig(hidden_size=128, num_hidden_layers=2, num_attention_heads=2, intermediate_size=256,
                                       num_register_tokens=4, patch_size=16, image_size=64, layer_norm_eps=1e-5,
                                       key_bias=False, query_bias=True, value_bias=True, proj_bias=True, mlp_bias=True,
                                       hidden_act="gelu", use_gated_mlp=False, layerscale_value=1.0, rope_theta=100.0,
                                       attention_dropout=0.0, drop_path_rate=0.0)
    model = transformers.DINOv3ViTModel(cfg)
    model.eval()
    # non-trivial values everywhere (HF init leaves biases at 0 and LayerScale at layerscale_value)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if "lambda1" in n:
                p.copy_(0.5 + torch.rand(p.shape, generator=g))
            elif n.endswith("bias") or "token" in n:
                p.copy_(torch.randn(p.shape, generator=g) * 0.05)
            elif "norm" in n and n.endswith("weight"):
                p.copy_(1.0 + 0.1 * torch.randn(p.shape, generator=g))
        for n, p in model.named_parameters():      # int8 * 2^e, exactly representable in float32 (and float64)
            scale = 2.0 ** math.ceil(math.log2(max(p.abs().max().item(), 1e-30) / 127))
            q = torch.round(p / scale).clamp(-127, 127)
            p.copy_(q * scale)
    arrays = {"meta": np.array([128, 2, 2, 16, 256, 4], dtype=np.int64)}
    for i, (H, W) in enumerate(SIZES):
        x = torch.randn(2, 3, H, W, generator=g).half().float()
        with torch.no_grad():
            out = model(pixel_values=x, output_hidden_states=True)
        arrays[f"x{i}"] = x.half().numpy()
        arrays[f"last{i}"] = out.last_hidden_state.numpy()
        arrays[f"hidden{i}"] = torch.stack(list(out.hidden_states)).numpy()   # [depth + 1, B, tokens, C]
    for k, v in model.state_dict().items():
        v = v.detach().float()
        scale = 2.0 ** math.ceil(math.log2(max(v.abs().max().item(), 1e-30) / 127))
        q = torch.round(v / scale)
        assert torch.equal(q * scale, v) and q.abs().max() <= 127
        arrays["hf:" + k] = q.to(torch.int8).numpy()
        arrays["scale:" + k] = np.float32(scale)
    path = os.path.join(HERE, "vit_hf_dinov3.npz")
    np.savez_compressed(path, **arrays)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB", "transformers", transformers.__version__)


if __name__ == "__main__":
    make()
