"""Drop-in for dvt/models/online_denoiser.py of the reference (SURVEY.md section 8(f-4), denoised-backbone inference):
same `Denoiser` constructor, parameters and state-dict names (`denoiser.*` with timm `Block` names, `pos_embed`, `vit.*`),
same `forward` flags and return values (online_denoiser.py:13-104).  The forward runs on the hand-written sm_90a kernels
of libdvt_b200.so: the frozen ViT through `PretrainedViTWrapper`, the learnable position embedding (resampled like
timm's `resample_abs_pos_embed` when the grid differs), then the denoiser block(s) as
LayerNorm -> QKV GEMM -> flash attention -> out-proj GEMM (+ residual) -> LayerNorm -> fc1 GEMM + GELU -> fc2 GEMM
(+ residual), no LayerScale (`init_values=None`).

TRAINING (SURVEY 8(f-2), reference main_denoiser.py:213-220): when gradients are enabled and the denoiser's parameters
require them, every block runs as ONE autograd node (`dvt.train_ops.block_forward`) whose backward is hand-written too:
flash-attention backward on wgmma, LayerNorm / GELU / bias gradients, bf16 data- and weight-gradient GEMMs that read
weights and activations in place as MN-major operands.  The position embedding (and its resampling, when the grid
differs) stays an ordinary torch op in the graph, so `pos_embed.grad` comes out of autograd."""
from __future__ import annotations

from typing import Dict, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import ops, train_ops
from .._lib import DvtError
from .vit_wrapper import PretrainedViTWrapper, _Block


class CenterPadding(nn.Module):
    """Zero-pads the trailing (spatial) dimensions of [B, C, ...] up to the next multiple of `multiple`, the surplus split
    evenly with the odd pixel on the far side -- what the dense-task evaluation puts in front of a denoised backbone so
    that any frame size maps onto whole patches (reference evaluation/eval_utils/misc.py:19-35)."""

    def __init__(self, multiple: int):
        super().__init__()
        self.multiple = int(multiple)

    def extra(self, size: int):
        total = -size % self.multiple
        return total // 2, total - total // 2

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        pads = []
        for dim in range(x.dim() - 1, 1, -1):       # F.pad lists the last dimension first
            pads.extend(self.extra(x.shape[dim]))
        return F.pad(x, pads)


class Denoiser(nn.Module):
    def __init__(self, noise_map_height: int = 37, noise_map_width: int = 37, feat_dim: int = 768,
                 vit: Optional[PretrainedViTWrapper] = None, enable_pe: bool = True, num_blocks: int = 1):
        super().__init__()
        assert feat_dim % 64 == 0, "the attention kernel needs head_dim 64 (reference: num_heads = feat_dim // 64)"
        self.vit = vit
        self.feat_dim, self.num_heads = feat_dim, feat_dim // 64
        self.noise_map_size = (noise_map_height, noise_map_width)
        mk = lambda: _Block(feat_dim, self.num_heads, 4 * feat_dim, swiglu=False, ls=False)  # noqa: E731
        self.denoiser = mk() if num_blocks <= 1 else nn.Sequential(*[mk() for _ in range(num_blocks)])
        self.pos_embed = None
        if enable_pe:
            self.pos_embed = nn.Parameter(torch.randn(1, noise_map_height * noise_map_width, feat_dim) * 0.02)
        if self.vit is not None:
            for p in self.vit.parameters():
                p.requires_grad = False
        self._wcache: Dict[int, tuple] = {}

    # ---- helpers ------------------------------------------------------------------------------------------------
    def _blocks(self):
        return list(self.denoiser) if isinstance(self.denoiser, nn.Sequential) else [self.denoiser]

    def _weights(self, blk: _Block):
        """bf16 copies of the GEMM weights, refreshed when a parameter changes (load_state_dict, optimiser step)."""
        ps = (blk.attn.qkv.weight, blk.attn.proj.weight, blk.mlp.fc1.weight, blk.mlp.fc2.weight)
        ver = tuple((p._version, p.data_ptr()) for p in ps)
        hit = self._wcache.get(id(blk))
        if hit is None or hit[0] != ver:
            hit = (ver, tuple(p.detach().to(torch.bfloat16).contiguous() for p in ps))
            self._wcache[id(blk)] = hit
        return hit[1]

    def _pos(self, h: int, w: int) -> Optional[torch.Tensor]:
        if self.pos_embed is None:
            return None
        pos = self.pos_embed.detach().float()
        gh, gw = self.noise_map_size
        if (h, w) != (gh, gw):   # timm.layers.resample_abs_pos_embed(num_prefix_tokens=0): bicubic, antialias, fp32
            g = pos.reshape(1, gh, gw, -1).permute(0, 3, 1, 2)
            g = F.interpolate(g, size=(h, w), mode="bicubic", antialias=True)
            pos = g.permute(0, 2, 3, 1).reshape(1, h * w, -1)
        return pos

    def _block_forward(self, x: torch.Tensor, blk: _Block, B: int, N: int) -> torch.Tensor:
        """x fp32 [B*N, C], updated in place (the residual stream), one pre-LN block without LayerScale."""
        wq, wp, w1, w2 = self._weights(blk)
        f32 = lambda t: t.detach().float().contiguous()  # noqa: E731
        xn = ops.layernorm(x, f32(blk.norm1.weight), f32(blk.norm1.bias), 1e-6, out_dtype=torch.bfloat16)
        qkv = ops.gemm_tn(xn, wq, f32(blk.attn.qkv.bias), None, torch.bfloat16)
        att = ops.attention(qkv.view(B, N, -1), self.num_heads).view(B * N, -1)
        ops.gemm_tn_residual_(x, att, wp, f32(blk.attn.proj.bias), None)
        xn = ops.layernorm(x, f32(blk.norm2.weight), f32(blk.norm2.bias), 1e-6, out_dtype=torch.bfloat16)
        hid = ops.gemm_tn(xn, w1, f32(blk.mlp.fc1.bias), "gelu", torch.bfloat16)
        ops.gemm_tn_residual_(x, hid, w2, f32(blk.mlp.fc2.bias), None)
        return x

    # ---- forward (online_denoiser.py:62-104) ----------------------------------------------------------------------
    def _wants_grad(self) -> bool:
        return torch.is_grad_enabled() and (any(p.requires_grad for p in self.denoiser.parameters())
                                            or (self.pos_embed is not None and self.pos_embed.requires_grad))

    def _pos_train(self, h: int, w: int) -> Optional[torch.Tensor]:
        """Position embedding inside the autograd graph (training): the parameter itself, or its bicubic resampling."""
        if self.pos_embed is None:
            return None
        gh, gw = self.noise_map_size
        if (h, w) == (gh, gw):
            return self.pos_embed.float()
        g = self.pos_embed.float().reshape(1, gh, gw, -1).permute(0, 3, 1, 2)
        g = train_ops.resample_bicubic(g, h, w)
        return g.permute(0, 2, 3, 1).reshape(1, h * w, -1)

    def forward(self, x, return_dict=False, return_channel_first=False, return_class_token=False, norm=True):
        class_tokens = None
        with torch.no_grad():
            if self.vit is not None:
                outs = self.vit.get_intermediate_layers(x, n=[self.vit.last_layer_index],
                                                        return_prefix_tokens=return_class_token, norm=norm)
                if return_class_token:
                    outs = outs[-1]
                    class_tokens = outs[1][:, 0]
                original_feats = outs[0].permute(0, 2, 3, 1)
                x = original_feats
            else:
                if not x.is_cuda:
                    raise DvtError("dvt_b200 Denoiser needs CUDA tensors (no CPU fallback)")
                original_feats = x.detach().clone()
        b, h, w, c = x.shape
        if self._wants_grad():
            # ---- training: one autograd node per block ----
            t = x.reshape(b, h * w, c).float()
            pos = self._pos_train(h, w)
            if pos is not None:
                t = t + pos
            t = t.reshape(b * h * w, c)
            for blk in self._blocks():
                t = train_ops.block_forward(t, blk, self.num_heads, b)
            out = t.reshape(b, h, w, c)
        else:
            with torch.no_grad():
                t = x.reshape(b, h * w, c).float()
                pos = self._pos(h, w)
                t = (t + pos) if pos is not None else t.clone()
                t = t.reshape(b * h * w, c).contiguous()
                for blk in self._blocks():
                    t = self._block_forward(t, blk, b, h * w)
                out = t.reshape(b, h, w, c)
        if return_channel_first:
            out = out.permute(0, 3, 1, 2)
        if return_dict:
            return {"denoised_feats": out, "original_feats": original_feats.detach(),
                    "class_tokens": class_tokens.detach() if class_tokens is not None else None}
        if return_class_token:
            assert class_tokens is not None
            return out, class_tokens
        return out
