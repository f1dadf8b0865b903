"""Backbone and head of the segmentation probe (reference evaluate_dense_tasks.py:177-214, evaluation/eval_utils/misc.py:38-88,
evaluation/segmentation/models/decode_heads/linear_head.py).

The backbone is frozen and in eval mode, and its input is zero-padded to whole patches (`CenterPadding(patch)`, the
forward pre-hook of the reference).  A ViT gives the timm model's own `get_intermediate_layers(n=out_indices,
reshape=True)` (misc.py:53-77 binds `backbone_model.model.get_intermediate_layers`), whose `norm` defaults to False in
timm 1.0.7: the blocks' outputs WITHOUT the final LayerNorm.  A Denoiser gives `[denoiser(x)] * 4` (its forward does
apply the final norm before the denoiser blocks).  The BNHead then keeps only the entries `in_index` selects, so
`ProbeBackbone` asks for the selected layers only, all of them from one pass over the blocks
(`forward_layers_concat`), written side by side in channels as `resize_concat` concatenates them: the same tensors, and
for the four-layer head (in_index [0, 1, 2, 3] of out_indices [8, 9, 10, 11]) 12 blocks instead of 9 + 10 + 11 + 12."""
from __future__ import annotations

import logging
import re
from typing import List, Optional, Sequence

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..models import CenterPadding, Denoiser, PretrainedViTWrapper

logger = logging.getLogger(__name__)


def build_backbone(backbone_type: str, load_distilled_model_from: Optional[str] = None,
                   load_denoiser_from: Optional[str] = None, num_blocks: int = 1, device="cuda") -> nn.Module:
    """evaluate_dense_tasks.py:177-214: the wrapper at stride = patch size, optionally with distilled weights (key
    "model", else "denoiser"), optionally under a Denoiser (noise map 37 at patch 14, 32 at patch 16) whose checkpoint
    "denoiser" is loaded with strict=False."""
    stride = int(re.search(r"patch(\d+)", backbone_type).group(1))
    vit = PretrainedViTWrapper(model_identifier=backbone_type, stride=stride).to(device)
    if load_distilled_model_from is not None:
        ckpt = torch.load(load_distilled_model_from, map_location="cpu")
        try:
            msg = vit.load_state_dict(ckpt["model"])
        except (KeyError, RuntimeError):
            msg = vit.load_state_dict(ckpt["denoiser"])
        logger.info("Loaded distilled model from %s (missing %s, unexpected %s)", load_distilled_model_from,
                    msg.missing_keys, msg.unexpected_keys)
    model: nn.Module = vit
    if load_denoiser_from is not None:
        pos_h = {14: 37, 16: 32}.get(stride)
        if pos_h is None:
            raise NotImplementedError(f"--load-denoiser-from: no noise-map size for patch {stride} (the reference knows "
                                      "14 and 16)")
        model = Denoiser(noise_map_height=pos_h, noise_map_width=pos_h, feat_dim=vit.n_output_dims, vit=vit,
                         num_blocks=num_blocks)
        msg = model.load_state_dict(torch.load(load_denoiser_from, map_location="cpu")["denoiser"], strict=False)
        logger.info("Loaded denoiser from %s (missing %s, unexpected %s)", load_denoiser_from,
                    {k for k in msg.missing_keys if "vit.model" not in k}, msg.unexpected_keys)
        model = model.to(device)
    for p in model.parameters():
        p.requires_grad = False
    return model.eval()


class ProbeBackbone(nn.Module):
    """Frozen feature extractor of the probe: x [B, 3, H, W] -> NHWC [B, h, w, C * len(in_index)] (the `resize_concat`
    input of the BNHead; the selected maps all share one grid, so the resize is the identity).

    A ViT's maps come from `forward_layers_concat` (one pass, the maps written side by side; bit for bit the maps of
    `get_intermediate_layers`).  The depth probe (`return_cls=True`, `norm=final_norm`) also takes prefix token 0 (the
    cls token, registers or not) of each layer from it, and the Denoiser's `denoiser(x, return_class_token=True,
    norm=norm)`, and returns (features, cls [B, C * len(in_index)])."""

    def __init__(self, model: nn.Module, out_indices: Sequence[int], in_index: Sequence[int], return_cls: bool = False,
                 norm: bool = False):
        super().__init__()
        self.model = model
        self.return_cls, self.norm = return_cls, norm
        self.is_denoiser = isinstance(model, Denoiser)
        vit = model.vit if self.is_denoiser else model
        self.pad = CenterPadding(vit.model.patch_embed.patch_size[0])
        self.in_index = list(in_index)
        self.layers = [list(out_indices)[i] for i in self.in_index]
        self.channels = vit.n_output_dims * len(self.in_index)

    @torch.no_grad()
    def forward(self, x: torch.Tensor):
        x = self.pad(x)
        if not self.is_denoiser:
            return self.model.model.forward_layers_concat(x, self.layers, norm=self.norm, return_cls=self.return_cls)
        if self.return_cls:
            f, c = self.model(x, return_class_token=True, norm=self.norm)
            if len(self.in_index) == 1:
                return f, c
            return torch.cat([f] * len(self.in_index), dim=-1), torch.cat([c] * len(self.in_index), dim=-1)
        f = self.model(x)                                      # [B, h, w, C]
        return f if len(self.in_index) == 1 else torch.cat([f] * len(self.in_index), dim=-1)


class LinearSegHead(nn.Module):
    """mmseg BNHead (linear_head.py): BatchNorm over the C channels (SyncBatchNorm under DDP), dropout 0, then the 1x1
    conv `conv_seg` C -> K (init normal std 0.01, bias 0).  Parameter names are those of the mmseg head, so the
    checkpoint's `decode_head.*` keys match.  Takes and returns NHWC: [B, h, w, C] -> [B, h, w, K]."""

    def __init__(self, channels: int, num_classes: int):
        super().__init__()
        self.bn = nn.BatchNorm2d(channels)
        self.conv_seg = nn.Conv2d(channels, num_classes, kernel_size=1)
        nn.init.normal_(self.conv_seg.weight, mean=0.0, std=0.01)
        nn.init.zeros_(self.conv_seg.bias)

    def forward(self, feat_nhwc: torch.Tensor) -> torch.Tensor:
        x = self.bn(feat_nhwc.permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
        K, C = self.conv_seg.weight.shape[:2]
        return F.linear(x, self.conv_seg.weight.view(K, C), self.conv_seg.bias).contiguous()


def head_state_dict(head: nn.Module) -> dict:
    return {"decode_head." + k: v for k, v in head.state_dict().items()}


def load_head_state_dict(head: nn.Module, sd: dict) -> None:
    head.load_state_dict({k[len("decode_head."):]: v for k, v in sd.items() if k.startswith("decode_head.")})


def in_channels_of(head_cfg: dict) -> List[int]:
    c = head_cfg.get("in_channels")
    return list(c) if isinstance(c, (list, tuple)) else [c]
