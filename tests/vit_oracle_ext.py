"""Oracle extension for the backbones built with timm `pre_norm=True` (the CLIP towers) and for head_dim 80 (ViT-H/14
MAE): CPU fp32, built on oracle/vit.py, whose functions it reuses unchanged.  Test infrastructure only.

  * patch_bias=False: timm passes `bias=not pre_norm` to the patch embedding, so the CLIP checkpoints have no
    `patch_embed.proj.bias`.
  * pre_norm=True: a LayerNorm `norm_pre` over the assembled tokens (cls + position) before the first block.
  * eps: every LayerNorm of the CLIP towers uses 1e-5 (timm `norm_layer=nn.LayerNorm`).
  * head_dim 80 needs nothing new: oracle.vit.attention derives head_dim from embed_dim / num_heads.

Pinned by tests/test_backbones_cpu.py against transformers.CLIPVisionModel and transformers.ViTModel (head_dim 80),
tests/golden/make_vit_golden_clip_hd80.py.  `embed` and `block` stay differentiable (the stage-3 gradient tests run
autograd through them).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, List, Sequence

import torch
import torch.nn.functional as F

from oracle import vit as OV


@dataclass
class ViTConfig(OV.ViTConfig):
    pre_norm: bool = False         # timm pre_norm=True: norm_pre LayerNorm before the blocks
    patch_bias: bool = True        # False: Conv2d patch embedding without bias


# timm 1.0.7 definitions of the three backbones (vision_transformer.py: vit_base_patch16_clip_{224,384} with
# pre_norm=True, norm_layer=nn.LayerNorm; vit_huge_patch14_224 with MAE weights).
CONFIGS: Dict[str, ViTConfig] = {
    "vit_base_patch16_clip_384.laion2b_ft_in12k_in1k": ViTConfig(768, 12, 12, 16, 384, 3072, layerscale=False, ln_eps=1e-5,
                                                                 pre_norm=True, patch_bias=False),
    "vit_base_patch16_clip_224.openai": ViTConfig(768, 12, 12, 16, 224, 3072, layerscale=False, ln_eps=1e-5, pre_norm=True,
                                                  patch_bias=False),
    "vit_huge_patch14_224.mae": ViTConfig(1280, 32, 16, 14, 224, 5120, layerscale=False),
}


def random_state_dict(cfg: ViTConfig, seed: int = 0, layerscale_range=(0.5, 1.5)) -> Dict[str, torch.Tensor]:
    """oracle.vit.random_state_dict plus norm_pre (pre_norm) and without the patch bias (patch_bias=False)."""
    sd = OV.random_state_dict(cfg, seed, layerscale_range)
    if not cfg.patch_bias:
        del sd["patch_embed.proj.bias"]
    if cfg.pre_norm:
        g = torch.Generator().manual_seed(seed + 7919)
        sd["norm_pre.weight"] = 1.0 + 0.1 * torch.randn(cfg.embed_dim, generator=g)
        sd["norm_pre.bias"] = 0.1 * torch.randn(cfg.embed_dim, generator=g)
    return sd


def embed(sd, cfg: ViTConfig, x: torch.Tensor, stride: int) -> torch.Tensor:
    """Token assembly of timm 1.0.7 (`patch_embed`, `_pos_embed`) followed by `norm_pre` when pre_norm."""
    if not cfg.patch_bias:
        assert "patch_embed.proj.bias" not in sd
        sd = dict(sd)
        sd["patch_embed.proj.bias"] = None  # F.conv2d without bias
    t = OV.embed(sd, cfg, x, stride)
    if cfg.pre_norm:
        t = F.layer_norm(t, (cfg.embed_dim,), sd["norm_pre.weight"], sd["norm_pre.bias"], cfg.ln_eps)
    return t


block = OV.block
feat_size = OV.feat_size


@torch.no_grad()
def forward_intermediates(sd, cfg: ViTConfig, x: torch.Tensor, indices: Sequence[int], stride: int | None = None,
                          norm: bool = True, reshape: bool = True, return_prefix_tokens: bool = False) -> List[torch.Tensor]:
    """oracle.vit.forward_intermediates with this module's `embed`."""
    stride = cfg.patch_size if stride is None else stride
    B, _, H, W = x.shape
    h, w = feat_size(cfg, H, W, stride)
    t = embed(sd, cfg, x.float(), stride)
    outs = []
    for i in range(max(indices) + 1):
        t = block(t, sd, i, cfg)
        if i in indices:
            outs.append(F.layer_norm(t, (cfg.embed_dim,), sd["norm.weight"], sd["norm.bias"], cfg.ln_eps) if norm else t)
    res = []
    for y in outs:
        prefix, feat = y[:, :cfg.num_prefix], y[:, cfg.num_prefix:]
        if reshape:
            feat = feat.reshape(B, h, w, -1).permute(0, 3, 1, 2).contiguous()
        res.append((feat, prefix) if return_prefix_tokens else feat)
    return res

