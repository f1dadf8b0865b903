"""Oracle extension for the DINOv3 backbones (2-D RoPE, registers, no absolute position embedding): CPU, any float dtype,
built on oracle/vit.py, whose functions it reuses unchanged.  Test infrastructure only.

RoPE as transformers `DINOv3ViTRopePositionEmbedding` computes it in eval mode:
  * inv_freq = 1 / base ** arange(0, 1, 4 / head_dim)   (base 100, head_dim 64: 16 frequencies)
  * patch centres of the token grid (h, w): ((i + 0.5) / h, (j + 0.5) / w) mapped to [-1, 1], rows in raster order
  * angles = 2 pi coord (x) inv_freq, flattened y-then-x (32 values) and tiled twice (64); cos / sin in fp32
  * q, k of the PATCH tokens only: q cos + rotate_half(q) sin, rotate_half(q) = cat(-q[32:], q[:32]) per head
The grid is the wrapper's ((H - P) // s + 1, (W - P) // s + 1).  At stride = patch it is HF's (H // P, W // P), which the
golden pins (tests/golden/make_vit_golden_dinov3.py -> vit_hf_dinov3.npz); at stride < patch this module DEFINES the
extension (same formula on the denser grid): no second implementation exists for it.

The state dict is the wrapper's container layout (timm-like names, `attn.qkv` with a zero k-bias slice, no pos_embed);
`embed` and `block` stay differentiable (the stage-3 gradient tests run autograd through them).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, List, Sequence, Tuple

import torch
import torch.nn.functional as F

from oracle import vit as OV


@dataclass
class RopeViTConfig(OV.ViTConfig):
    rope_base: float = 100.0


# the three DINOv3 LVD-1689M backbones (width / depth / heads, MLP ratio 4, patch 16, 4 registers, LayerNorm eps 1e-5)
CONFIGS: Dict[str, RopeViTConfig] = {
    f"vit_{n}_patch16_dinov3.lvd1689m": RopeViTConfig(C, d, hd, 16, 224, 4 * C, num_reg_tokens=4, no_embed_class=True,
                                                      ln_eps=1e-5)
    for n, C, d, hd in (("small", 384, 12, 6), ("base", 768, 12, 12), ("large", 1024, 24, 16))
}


def rope_cos_sin(h: int, w: int, head_dim: int = 64, base: float = 100.0) -> Tuple[torch.Tensor, torch.Tensor]:
    """(cos, sin) fp32 [h * w, head_dim] of the token grid (h, w)."""
    inv_freq = 1.0 / base ** torch.arange(0, 1, 4 / head_dim, dtype=torch.float32)
    ch = torch.arange(0.5, h, dtype=torch.float32) / h
    cw = torch.arange(0.5, w, dtype=torch.float32) / w
    coords = torch.stack(torch.meshgrid(ch, cw, indexing="ij"), dim=-1).flatten(0, 1)
    coords = 2.0 * coords - 1.0
    angles = (2 * math.pi * coords[:, :, None] * inv_freq[None, None, :]).flatten(1, 2).tile(2)
    return torch.cos(angles), torch.sin(angles)


def rotate_half(x: torch.Tensor) -> torch.Tensor:
    x1, x2 = x[..., : x.shape[-1] // 2], x[..., x.shape[-1] // 2:]
    return torch.cat((-x2, x1), dim=-1)


def apply_rope(t: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, prefix: int) -> torch.Tensor:
    """t [B, heads, N, 64]: rotates the rows >= prefix (patch tokens), leaves the prefix rows as they are."""
    pre, pat = t[:, :, :prefix], t[:, :, prefix:]
    cos, sin = cos.to(t.dtype), sin.to(t.dtype)
    return torch.cat([pre, pat * cos + rotate_half(pat) * sin], dim=2)


def attention(x, qkv_w, qkv_b, proj_w, proj_b, num_heads: int, cos, sin, prefix: int) -> torch.Tensor:
    B, N, C = x.shape
    hd = C // num_heads
    qkv = F.linear(x, qkv_w, qkv_b).reshape(B, N, 3, num_heads, hd).permute(2, 0, 3, 1, 4)
    q, k, v = qkv.unbind(0)
    q, k = apply_rope(q, cos, sin, prefix), apply_rope(k, cos, sin, prefix)
    attn = ((q * hd ** -0.5) @ k.transpose(-2, -1)).softmax(dim=-1)
    out = (attn @ v).transpose(1, 2).reshape(B, N, C)
    return F.linear(out, proj_w, proj_b)


def block(x: torch.Tensor, sd, i: int, cfg: RopeViTConfig, cos, sin) -> torch.Tensor:
    """oracle.vit.block with the rotary attention."""
    p = f"blocks.{i}."
    C = cfg.embed_dim
    y = F.layer_norm(x, (C,), sd[p + "norm1.weight"], sd[p + "norm1.bias"], cfg.ln_eps)
    y = attention(y, sd[p + "attn.qkv.weight"], sd[p + "attn.qkv.bias"], sd[p + "attn.proj.weight"], sd[p + "attn.proj.bias"],
                  cfg.num_heads, cos, sin, cfg.num_prefix)
    if cfg.layerscale:
        y = y * sd[p + "ls1.gamma"]
    x = x + y
    y = F.layer_norm(x, (C,), sd[p + "norm2.weight"], sd[p + "norm2.bias"], cfg.ln_eps)
    y = OV.mlp(y, sd, p, cfg)
    if cfg.layerscale:
        y = y * sd[p + "ls2.gamma"]
    return x + y


def embed(sd, cfg: RopeViTConfig, x: torch.Tensor, stride: int) -> torch.Tensor:
    """Patch embedding with the overridden stride, then [cls, registers, patches]; no position term."""
    B = x.shape[0]
    t = F.conv2d(x, sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=stride)
    t = t.flatten(2).transpose(1, 2)
    return torch.cat([sd["cls_token"].expand(B, -1, -1), sd["reg_token"].expand(B, -1, -1), t], dim=1)


def hidden_states(sd, cfg: RopeViTConfig, x: torch.Tensor, stride: int | None = None) -> List[torch.Tensor]:
    """[token assembly, output of block 0, ..., output of the last block] (HF `output_hidden_states`)."""
    stride = cfg.patch_size if stride is None else stride
    h, w = OV.feat_size(cfg, x.shape[2], x.shape[3], stride)
    cos, sin = rope_cos_sin(h, w, cfg.embed_dim // cfg.num_heads, cfg.rope_base)
    t = embed(sd, cfg, x, stride)
    outs = [t]
    for i in range(cfg.depth):
        t = block(t, sd, i, cfg, cos, sin)
        outs.append(t)
    return outs


@torch.no_grad()
def forward_intermediates(sd: Dict[str, torch.Tensor], cfg: RopeViTConfig, x: torch.Tensor, indices: Sequence[int],
                          stride: int | None = None, norm: bool = True, reshape: bool = True,
                          return_prefix_tokens: bool = False) -> List[torch.Tensor]:
    """`PretrainedViTWrapper.get_intermediate_layers(x, n=indices, reshape, return_prefix_tokens, norm)` of a DINOv3 ViT;
    computes in the dtype of `x` and `sd` (float64 for the golden comparison)."""
    stride = cfg.patch_size if stride is None else stride
    B = x.shape[0]
    h, w = OV.feat_size(cfg, x.shape[2], x.shape[3], stride)
    cos, sin = rope_cos_sin(h, w, cfg.embed_dim // cfg.num_heads, cfg.rope_base)
    t = embed(sd, cfg, x, stride)
    res = []
    for i in range(max(indices) + 1):
        t = block(t, sd, i, cfg, cos, sin)
        if i in indices:
            y = F.layer_norm(t, (cfg.embed_dim,), sd["norm.weight"], sd["norm.bias"], cfg.ln_eps) if norm else t
            prefix, feat = y[:, :cfg.num_prefix], y[:, cfg.num_prefix:]
            if reshape:
                feat = feat.reshape(B, h, w, -1).permute(0, 3, 1, 2).contiguous()
            res.append((feat, prefix) if return_prefix_tokens else feat)
    return res


def load_golden(path: str):
    """tests/golden/vit_hf_dinov3.npz -> (npz, HF-layout float32 state dict, [x0, x1] float32): the int8 parameters times
    their power-of-two scales and the float16 inputs, i.e. exactly the values transformers ran with."""
    import numpy as np
    z = np.load(path)
    hf = {k[3:]: torch.from_numpy(z[k].astype(np.float32) * z["scale:" + k[3:]]) for k in z.files if k.startswith("hf:")}
    xs = [torch.from_numpy(z[f"x{i}"].astype(np.float32)) for i in (0, 1)]
    return z, hf, xs


def random_state_dict(cfg: RopeViTConfig, seed: int = 0) -> Dict[str, torch.Tensor]:
    """oracle.vit.random_state_dict in the DINOv3 container layout: no pos_embed, k-bias slice of attn.qkv zero."""
    sd = OV.random_state_dict(cfg, seed)
    del sd["pos_embed"]
    C = cfg.embed_dim
    for i in range(cfg.depth):
        sd[f"blocks.{i}.attn.qkv.bias"][C:2 * C] = 0
    return sd
