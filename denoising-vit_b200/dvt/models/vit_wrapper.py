"""Drop-in for dvt/models/vit_wrapper.py of the reference: same `MODEL_LIST`, same `PretrainedViTWrapper`
constructor, attributes and `get_intermediate_layers` contract (reference vit_wrapper.py:15-146), with the forward
executed by libdvt_b200.so (hand-written sm_90a kernels) instead of timm.

Training (stage 3, reference main_distillation.py): after `set_trainable()`, calls made with gradients enabled return a
differentiable result whose backward is hand-written CUDA too (dvt.train_ops: patch embedding, pre-LN blocks with
LayerScale and a GELU or SwiGLU MLP, final norm with the prefix strip); `set_grad_checkpointing(True)` makes every block recompute its forward in
the backward instead of keeping its activations.  Without `set_trainable()` every call is the inference forward.

`self.model` is a parameter container whose state-dict keys are timm's, so checkpoints of the wrapper
(`model.<timm key>`, reference make_video_demo.py:31-34) load unchanged.  There is no network in this build:
`pretrained=True` weights are read from `$DVT_WEIGHTS_DIR/<model_identifier>.pth` when present, otherwise the
model is randomly initialised (timm-style) and a warning is logged.
"""
from __future__ import annotations

import logging
import math
import os
import re
from ctypes import byref, c_int, c_void_p
from typing import List, Optional, Tuple, Union

import torch
import torch.nn.functional as F
from torch import nn

from .. import _lib, train_ops
from .._lib import check, cur_stream, lib, ptr

logger = logging.getLogger(__name__)

# Same list as the reference (vit_wrapper.py:15-56); argparse `choices` in the stage-1/2 CLIs depend on it.
MODEL_LIST = [
    "vit_small_patch8_224.dino",
    "vit_small_patch16_224.dino",
    "vit_base_patch8_224.dino",
    "vit_base_patch16_224.dino",
    "vit_small_patch14_dinov2.lvd142m",
    "vit_base_patch14_dinov2.lvd142m",
    "vit_large_patch14_dinov2.lvd142m",
    "vit_giant_patch14_dinov2.lvd142m",
    "vit_small_patch14_reg4_dinov2.lvd142m",
    "vit_base_patch14_reg4_dinov2.lvd142m",
    "vit_large_patch14_reg4_dinov2.lvd142m",
    "vit_giant_patch14_reg4_dinov2.lvd142m",
    "vit_base_patch16_224.mae",
    "vit_large_patch16_224.mae",
    "vit_huge_patch14_224.mae",
    "vit_base_patch16_clip_384.laion2b_ft_in12k_in1k",
    "vit_base_patch16_clip_224.openai",
    "eva02_base_patch16_clip_224.merged2b",
    "deit3_base_patch16_224.fb_in1k",
    "vit_base_patch16_384.augreg_in21k_ft_in1k",
]
# DINOv3 (LVD-1689M weights), after the reference's list: 2-D RoPE ViTs, DINOV3_ARCHS below
MODEL_LIST.extend([
    "vit_small_patch16_dinov3.lvd1689m",
    "vit_base_patch16_dinov3.lvd1689m",
    "vit_large_patch16_dinov3.lvd1689m",
])

IMAGENET_MEAN, IMAGENET_STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
HALF_MEAN, HALF_STD = (0.5, 0.5, 0.5), (0.5, 0.5, 0.5)
OPENAI_CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


def _arch(embed, depth, heads, img, mlp=None, swiglu=False, ls=False, reg=0, no_embed_class=False,
          mean=IMAGENET_MEAN, std=IMAGENET_STD, pre_norm=False, patch_bias=True, ln_eps=1e-6, rope=False):
    return dict(embed=embed, depth=depth, heads=heads, img=img, mlp=mlp or 4 * embed, swiglu=swiglu, ls=ls, reg=reg,
                no_embed_class=no_embed_class, mean=mean, std=std, pre_norm=pre_norm, patch_bias=patch_bias,
                ln_eps=ln_eps, rope=rope)


# Pre-LN ViTs with head_dim 64 or 80 (what the CUDA path implements).  The CLIP towers are timm's pre_norm=True,
# norm_layer=nn.LayerNorm build: a `norm_pre` LayerNorm before the first block, LayerNorm eps 1e-5, a patch embedding
# without bias, OpenAI CLIP normalisation; their MLP is erf GELU (timm 1.0.7 keeps QuickGELU to the separate
# *_clip_quickgelu_* models).  ViT-H/14 MAE has head_dim 1280 / 16 = 80.  EVA02 (2-D RoPE, SwiGLU with sub-LN, inner
# attention norm) is listed in MODEL_LIST for CLI compatibility but raises here (DESIGN.md section 8).
ARCHS = {
    "vit_small_patch8_224.dino": _arch(384, 12, 6, 224),
    "vit_small_patch16_224.dino": _arch(384, 12, 6, 224),
    "vit_base_patch8_224.dino": _arch(768, 12, 12, 224),
    "vit_base_patch16_224.dino": _arch(768, 12, 12, 224),
    "vit_small_patch14_dinov2.lvd142m": _arch(384, 12, 6, 518, ls=True),
    "vit_base_patch14_dinov2.lvd142m": _arch(768, 12, 12, 518, ls=True),
    "vit_large_patch14_dinov2.lvd142m": _arch(1024, 24, 16, 518, ls=True),
    "vit_giant_patch14_dinov2.lvd142m": _arch(1536, 40, 24, 518, mlp=8192, swiglu=True, ls=True),
    "vit_small_patch14_reg4_dinov2.lvd142m": _arch(384, 12, 6, 518, ls=True, reg=4, no_embed_class=True),
    "vit_base_patch14_reg4_dinov2.lvd142m": _arch(768, 12, 12, 518, ls=True, reg=4, no_embed_class=True),
    "vit_large_patch14_reg4_dinov2.lvd142m": _arch(1024, 24, 16, 518, ls=True, reg=4, no_embed_class=True),
    "vit_giant_patch14_reg4_dinov2.lvd142m": _arch(1536, 40, 24, 518, mlp=8192, swiglu=True, ls=True, reg=4,
                                                   no_embed_class=True),
    "vit_base_patch16_224.mae": _arch(768, 12, 12, 224),
    "vit_large_patch16_224.mae": _arch(1024, 24, 16, 224),
    "vit_huge_patch14_224.mae": _arch(1280, 32, 16, 224),
    "vit_base_patch16_clip_384.laion2b_ft_in12k_in1k": _arch(768, 12, 12, 384, mean=OPENAI_CLIP_MEAN, std=OPENAI_CLIP_STD,
                                                             pre_norm=True, patch_bias=False, ln_eps=1e-5),
    "vit_base_patch16_clip_224.openai": _arch(768, 12, 12, 224, mean=OPENAI_CLIP_MEAN, std=OPENAI_CLIP_STD, pre_norm=True,
                                              patch_bias=False, ln_eps=1e-5),
    "deit3_base_patch16_224.fb_in1k": _arch(768, 12, 12, 224, ls=True, no_embed_class=True),
    "vit_base_patch16_384.augreg_in21k_ft_in1k": _arch(768, 12, 12, 384, mean=HALF_MEAN, std=HALF_STD),
}

# DINOv3 ViT-S/B/L/16 (transformers DINOv3ViTModel): pre-LN blocks with LayerScale and a GELU MLP (ratio 4), LayerNorm eps
# 1e-5, 4 register tokens, no absolute position embedding but a 2-D RoPE on q and k of the patch tokens (rope=True: fused
# into the QKV GEMM epilogue, DESIGN.md section 8), q and v biases and no k bias (key_bias=False: the k slice of attn.qkv.bias
# stays zero, in training too), ImageNet normalisation.
DINOV3_ARCHS = {
    "vit_small_patch16_dinov3.lvd1689m": _arch(384, 12, 6, 224, ls=True, reg=4, no_embed_class=True, ln_eps=1e-5, rope=True),
    "vit_base_patch16_dinov3.lvd1689m": _arch(768, 12, 12, 224, ls=True, reg=4, no_embed_class=True, ln_eps=1e-5, rope=True),
    "vit_large_patch16_dinov3.lvd1689m": _arch(1024, 24, 16, 224, ls=True, reg=4, no_embed_class=True, ln_eps=1e-5,
                                               rope=True),
}

ROPE_BASE = 100.0   # DINOv3ViTConfig.rope_theta


def arch_of(identifier: str) -> dict:
    """The architecture entry of a backbone identifier, from ARCHS or DINOV3_ARCHS; NotImplementedError for the listed
    identifiers the H100 path does not run (EVA02)."""
    a = ARCHS.get(identifier) or DINOV3_ARCHS.get(identifier)
    if a is None:
        raise NotImplementedError(
            f"{identifier}: architecture outside the pre-LN ViT family (head_dim 64 / 80) is not "
            "implemented by the H100 path (see DESIGN.md, out of scope)")
    return a


def rope_table(h: int, w: int, head_dim: int = 64, base: float = ROPE_BASE) -> torch.Tensor:
    """f32 [h * w, head_dim] (CPU): row p = (cos | sin) of the head_dim / 2 angles of patch p on the token grid (h, w), as
    transformers DINOv3ViTRopePositionEmbedding computes them in eval mode: patch centres ((i + 0.5) / h, (j + 0.5) / w)
    mapped to [-1, 1], angles = 2 pi coord (x) inv_freq flattened y-then-x, inv_freq = 1 / base ** arange(0, 1, 4 /
    head_dim), all in fp32.  (HF tiles the angles twice; the kernels pair columns d and d + head_dim / 2 instead.)"""
    inv_freq = 1.0 / base ** torch.arange(0, 1, 4 / head_dim, dtype=torch.float32)
    ch = torch.arange(0.5, h, dtype=torch.float32) / h
    cw = torch.arange(0.5, w, dtype=torch.float32) / w
    coords = 2.0 * torch.stack(torch.meshgrid(ch, cw, indexing="ij"), dim=-1).flatten(0, 1) - 1.0
    angles = (2 * math.pi * coords[:, :, None] * inv_freq[None, None, :]).flatten(1, 2)
    return torch.cat([torch.cos(angles), torch.sin(angles)], dim=1).contiguous()


_HF_LAYER = re.compile(r"^(?:model\.)?layer\.(\d+)\.(.+)$")
_HF_BLOCK_KEYS = {"norm1.weight": "norm1.weight", "norm1.bias": "norm1.bias", "norm2.weight": "norm2.weight",
                  "norm2.bias": "norm2.bias", "attention.o_proj.weight": "attn.proj.weight",
                  "attention.o_proj.bias": "attn.proj.bias", "layer_scale1.lambda1": "ls1.gamma",
                  "layer_scale2.lambda1": "ls2.gamma", "mlp.up_proj.weight": "mlp.fc1.weight",
                  "mlp.up_proj.bias": "mlp.fc1.bias", "mlp.down_proj.weight": "mlp.fc2.weight",
                  "mlp.down_proj.bias": "mlp.fc2.bias"}


def is_hf_dinov3_state_dict(sd) -> bool:
    return any(k.startswith("embeddings.") for k in sd)


def hf_dinov3_to_container(sd) -> dict:
    """`DINOv3ViTModel.state_dict()` keys -> the container's (timm-like) keys: q / k / v projections stacked into attn.qkv
    with a zero k-bias slice (key_bias=False), LayerScale lambda1 -> gamma, up / down_proj -> fc1 / fc2; mask_token (a
    pretraining-only parameter) is dropped.  Accepts the layer keys with or without HF's `model.` prefix."""
    out, qkv = {}, {}
    for k, v in sd.items():
        if k == "embeddings.cls_token":
            out["cls_token"] = v
        elif k == "embeddings.register_tokens":
            out["reg_token"] = v
        elif k.startswith("embeddings.patch_embeddings."):
            out["patch_embed.proj." + k[len("embeddings.patch_embeddings."):]] = v
        elif k == "embeddings.mask_token":
            continue
        elif k in ("norm.weight", "norm.bias"):
            out[k] = v
        else:
            m = _HF_LAYER.match(k)
            if m is None:
                raise KeyError(f"unexpected key in a DINOv3 state dict: {k}")
            i, rest = int(m.group(1)), m.group(2)
            if rest.startswith("attention.") and rest[len("attention.")] in "qkv" and rest[len("attention.") + 1:].startswith("_proj."):
                qkv.setdefault(i, {})[rest[len("attention."):]] = v
            elif rest in _HF_BLOCK_KEYS:
                out[f"blocks.{i}.{_HF_BLOCK_KEYS[rest]}"] = v
            else:
                raise KeyError(f"unexpected key in a DINOv3 state dict: {k}")
    for i, d in qkv.items():
        out[f"blocks.{i}.attn.qkv.weight"] = torch.cat([d["q_proj.weight"], d["k_proj.weight"], d["v_proj.weight"]])
        out[f"blocks.{i}.attn.qkv.bias"] = torch.cat([d["q_proj.bias"], torch.zeros_like(d["q_proj.bias"]), d["v_proj.bias"]])
    return out


class _LayerScale(nn.Module):
    def __init__(self, dim, init=1e-5):
        super().__init__()
        self.gamma = nn.Parameter(init * torch.ones(dim))


class _Attn(nn.Module):
    def __init__(self, dim, heads):
        super().__init__()
        self.num_heads = heads
        self.qkv = nn.Linear(dim, 3 * dim)
        self.proj = nn.Linear(dim, dim)


class _Mlp(nn.Module):
    def __init__(self, dim, hidden, swiglu):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.fc2 = nn.Linear(hidden // 2 if swiglu else hidden, dim)


class _Block(nn.Module):
    def __init__(self, dim, heads, hidden, swiglu, ls, eps=1e-6):
        super().__init__()
        self.norm1 = nn.LayerNorm(dim, eps=eps)
        self.attn = _Attn(dim, heads)
        self.ls1 = _LayerScale(dim) if ls else nn.Identity()
        self.norm2 = nn.LayerNorm(dim, eps=eps)
        self.mlp = _Mlp(dim, hidden, swiglu)
        self.ls2 = _LayerScale(dim) if ls else nn.Identity()


class _PatchEmbed(nn.Module):
    def __init__(self, patch, dim, bias=True):
        super().__init__()
        self.patch_size = (patch, patch)
        self.proj = nn.Conv2d(3, dim, kernel_size=patch, stride=patch, bias=bias)

    def dynamic_feat_size(self, img_size: Tuple[int, int]) -> Tuple[int, int]:
        # reference vit_wrapper.py:81-87
        return ((img_size[0] - self.patch_size[0]) // self.proj.stride[0] + 1,
                (img_size[1] - self.patch_size[1]) // self.proj.stride[1] + 1)


class B200VisionTransformer(nn.Module):
    """Parameter container with timm's VisionTransformer attribute and state-dict names; the forward is CUDA.  A RoPE
    arch (DINOv3) has no pos_embed, and `load_state_dict` also takes transformers' DINOv3ViTModel layout."""

    def __init__(self, identifier: str, patch: int, a: dict):
        super().__init__()
        self.identifier = identifier
        self.arch = a
        dim = a["embed"]
        self.embed_dim = self.num_features = dim
        self.num_prefix_tokens = 1 + a["reg"]
        self.num_reg_tokens = a["reg"]
        self.no_embed_class = a["no_embed_class"]
        self.rope = bool(a.get("rope", False))
        self.dynamic_img_size = True
        grid = a["img"] // patch
        self.native_grid = (grid, grid)
        self.patch_embed = _PatchEmbed(patch, dim, bias=a["patch_bias"])
        self.cls_token = nn.Parameter(torch.zeros(1, 1, dim))
        if a["reg"]:
            self.reg_token = nn.Parameter(torch.zeros(1, a["reg"], dim))
        if not self.rope:
            n_pos = grid * grid + (0 if a["no_embed_class"] else 1)
            self.pos_embed = nn.Parameter(torch.randn(1, n_pos, dim) * 0.02)
        eps = a["ln_eps"]
        if a["pre_norm"]:  # timm pre_norm=True (CLIP): LayerNorm over the assembled tokens before the first block
            self.norm_pre = nn.LayerNorm(dim, eps=eps)
        self.blocks = nn.ModuleList([_Block(dim, a["heads"], a["mlp"], a["swiglu"], a["ls"], eps) for _ in range(a["depth"])])
        self.norm = nn.LayerNorm(dim, eps=eps)
        self._init_weights()
        self._handle: Optional[c_void_p] = None
        self._dirty = True
        self._pos_cache = {}
        self._param_sig = None
        self._trainable = False
        self._grad_ckpt = False

    def _init_weights(self):
        nn.init.normal_(self.cls_token, std=1e-6)
        if self.num_reg_tokens:
            nn.init.normal_(self.reg_token, std=1e-6)
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.trunc_normal_(m.weight, std=0.02)
                nn.init.zeros_(m.bias)

    def set_grad_checkpointing(self, enable: bool = True):
        """timm API: the blocks of the training path keep only their input and recompute the rest in the backward."""
        self._grad_ckpt = bool(enable)

    # ---- weight plumbing ------------------------------------------------------------------------------
    def _apply(self, fn, *a, **k):
        self._dirty = True
        self._pos_cache = {}
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, state_dict, *a, **k):
        if self.rope and is_hf_dinov3_state_dict(state_dict):
            state_dict = hf_dinov3_to_container(state_dict)
        self._dirty = True
        self._pos_cache = {}
        return super().load_state_dict(state_dict, *a, **k)

    def mark_dirty(self):
        """Call after editing parameters in place."""
        self._dirty = True
        self._pos_cache = {}

    def _sync(self):
        a = self.arch
        # parameters changed in place (an optimiser step; FusedAdamW also re-points them into its flat buffer): the
        # handle's bf16 copies and the cached position tables are stale
        sig = tuple((p._version, p.data_ptr()) for p in self.parameters())
        if sig != self._param_sig:
            self._dirty = True
            self._pos_cache = {}
        if self._handle is None:
            h = c_void_p()
            check(lib().dvt_vit_create(byref(h), a["embed"], a["depth"], a["heads"], self.patch_embed.patch_size[0],
                                       a["mlp"], int(a["swiglu"]), int(a["ls"]), self.num_prefix_tokens, a["ln_eps"],
                                       int(a["pre_norm"]), int(a["patch_bias"]), int(self.rope)), "dvt_vit_create")
            self._handle = h
        if not self._dirty:
            return
        skip = ("cls_token", "reg_token", "pos_embed")
        for k, v in self.state_dict().items():
            if k in skip:
                continue
            t = v.detach().to(dtype=torch.float32).contiguous()
            check(lib().dvt_vit_load(self._handle, k.encode(), ptr(t), t.numel()), f"dvt_vit_load({k})")
        self._dirty = False
        self._param_sig = sig

    def __del__(self):
        try:
            if self._handle is not None:
                lib().dvt_vit_destroy(self._handle)
        except Exception:
            pass

    def _rope_table(self, h: int, w: int, device) -> torch.Tensor:
        """The RoPE table f32 [h*w, 64] of the token grid (h, w) on `device` (`rope_table`), cached like the position
        tables."""
        key = ("rope", h, w, str(device))
        if key not in self._pos_cache:
            self._pos_cache[key] = rope_table(h, w, self.embed_dim // self.arch["heads"]).to(device)
        return self._pos_cache[key]

    def _pos_tables(self, h: int, w: int, device) -> Tuple[Optional[torch.Tensor], torch.Tensor]:
        """(pos_patch [h*w, C], prefix_rows [prefix, C]) following timm 1.0.7 `_pos_embed` + resample_abs_pos_embed
        (bicubic, antialias, fp32; reference restatement evaluation/vitdet/vision_transformer.py:120-138).  RoPE archs:
        (None, [cls, registers])."""
        key = (h, w, str(device))
        if key not in self._pos_cache and self.rope:
            with torch.no_grad():
                rows = [self.cls_token.detach().float().to(device)[0], self.reg_token.detach().float().to(device)[0]]
                self._pos_cache[key] = (None, torch.cat(rows, 0).contiguous())
        if key not in self._pos_cache:
            with torch.no_grad():
                pos = self.pos_embed.detach().float().to(device)
                npre = 0 if self.no_embed_class else 1
                pre, grid = pos[:, :npre], pos[:, npre:]
                gh, gw = self.native_grid
                if (h, w) != (gh, gw):
                    C = grid.shape[-1]
                    g = grid.reshape(1, gh, gw, C).permute(0, 3, 1, 2)
                    g = F.interpolate(g, size=(h, w), mode="bicubic", antialias=True)
                    grid = g.permute(0, 2, 3, 1).reshape(1, h * w, C)
                cls = self.cls_token.detach().float().to(device)[0]
                if not self.no_embed_class:
                    cls = cls + pre[0]
                rows = [cls]
                if self.num_reg_tokens:
                    rows.append(self.reg_token.detach().float().to(device)[0])
                self._pos_cache[key] = (grid[0].contiguous(), torch.cat(rows, 0).contiguous())
        return self._pos_cache[key]

    def _pos_tables_train(self, h: int, w: int) -> Tuple[Optional[torch.Tensor], torch.Tensor]:
        """`_pos_tables` inside the autograd graph: gradients reach pos_embed, cls_token and reg_token."""
        if self.rope:
            return None, torch.cat([self.cls_token.float()[0], self.reg_token.float()[0]], 0)
        pos = self.pos_embed.float()
        npre = 0 if self.no_embed_class else 1
        pre, grid = pos[:, :npre], pos[:, npre:]
        gh, gw = self.native_grid
        if (h, w) != (gh, gw):
            C = grid.shape[-1]
            g = grid.reshape(1, gh, gw, C).permute(0, 3, 1, 2)
            g = train_ops.resample_bicubic(g, h, w)
            grid = g.permute(0, 2, 3, 1).reshape(1, h * w, C)
        cls = self.cls_token.float()[0]
        if not self.no_embed_class:
            cls = cls + pre[0]
        rows = [cls]
        if self.num_reg_tokens:
            rows.append(self.reg_token.float()[0])
        return grid[0], torch.cat(rows, 0)

    def _training(self) -> bool:
        return self._trainable and torch.is_grad_enabled()

    def _run_train(self, x: torch.Tensor, layer_index: int, norm: bool) -> torch.Tensor:
        """Differentiable forward to the [B, h, w, C] map of `layer_index` (prefix tokens stripped)."""
        if not x.is_cuda:
            raise _lib.DvtError("dvt_b200 ViT training needs a CUDA tensor (no CPU fallback)")
        if x.dtype not in (torch.float32, torch.bfloat16):
            x = x.float()
        x = x.contiguous()
        B, _, H, W = x.shape
        P = self.patch_embed.patch_size[0]
        stride = int(self.patch_embed.proj.stride[0])
        h, w = (H - P) // stride + 1, (W - P) // stride + 1
        prefix, ntok, C = self.num_prefix_tokens, self.num_prefix_tokens + h * w, self.embed_dim
        pos_patch, prefix_rows = self._pos_tables_train(h, w)
        rope = (self._rope_table(h, w, x.device), prefix) if self.rope else None
        eps = self.arch["ln_eps"]
        t = train_ops.vit_embed(x, self.patch_embed.proj.weight, self.patch_embed.proj.bias, pos_patch, prefix_rows, stride)
        if self.arch["pre_norm"]:
            t = train_ops.vit_layernorm(t, self.norm_pre.weight, self.norm_pre.bias, eps)
        for i in range(layer_index + 1):
            t = train_ops.vit_block_forward(t, self.blocks[i], self.arch["heads"], B, checkpoint=self._grad_ckpt, eps=eps,
                                            rope=rope)
        if norm:
            y = train_ops.vit_norm_strip(t, self.norm.weight, self.norm.bias, ntok, prefix, eps)
        else:
            y = t.view(B, ntok, C)[:, prefix:]
        return y.reshape(B, h, w, C)

    # ---- forward --------------------------------------------------------------------------------------
    def _prep(self, x: torch.Tensor):
        """(x as a contiguous f32 / bf16 CUDA tensor, stride, h, w, pos_patch, prefix_rows, rope) of one inference forward,
        with the handle's weights up to date."""
        if not x.is_cuda:
            raise _lib.DvtError("dvt_b200 ViT forward needs a CUDA tensor (no CPU fallback)")
        if x.dtype not in (torch.float32, torch.bfloat16):
            x = x.float()
        x = x.contiguous()
        self._sync()
        _, _, H, W = x.shape
        P = self.patch_embed.patch_size[0]
        stride = int(self.patch_embed.proj.stride[0])
        h, w = (H - P) // stride + 1, (W - P) // stride + 1
        pos_patch, prefix_rows = self._pos_tables(h, w, x.device)
        rope = self._rope_table(h, w, x.device) if self.rope else None
        return x, stride, h, w, pos_patch, prefix_rows, rope

    def _run(self, x: torch.Tensor, layer_index: int, norm: bool, all_tokens: bool,
             out: Optional[torch.Tensor] = None) -> torch.Tensor:
        x, stride, h, w, pos_patch, prefix_rows, rope = self._prep(x)
        B, _, H, W = x.shape
        C = self.embed_dim
        shape = (B, self.num_prefix_tokens + h * w, C) if all_tokens else (B, h, w, C)
        if out is None:
            out = torch.empty(shape, device=x.device, dtype=torch.float32)
        else:  # caller-provided destination (e.g. a slice of the stage-1 feature bank)
            assert tuple(out.shape) == shape and out.dtype == torch.float32 and out.is_contiguous() and out.is_cuda
        check(lib().dvt_vit_forward(self._handle, ptr(x), 0 if x.dtype == torch.bfloat16 else 1, B, H, W, stride,
                                    ptr(pos_patch), ptr(prefix_rows), ptr(rope), layer_index, int(norm), ptr(out),
                                    int(all_tokens), cur_stream()), "dvt_vit_forward")
        return out

    def _run_layers(self, x: torch.Tensor, layers: List[int], norm: bool, all_tokens: bool = False, concat: bool = False,
                    prefix: bool = False):
        """One dvt_vit_forward_layers pass over `layers` (strictly ascending).  Returns (maps, prefix_rows): maps is one
        [B, h, w, L*C] tensor with the layers' maps side by side in channels (concat), else a list of one tensor per layer,
        [B, h, w, C] ([B, prefix + h*w, C] with all_tokens); prefix_rows is [L, B, prefix, C] (prefix) or None."""
        x, stride, h, w, pos_patch, prefix_rows, rope = self._prep(x)
        B, _, H, W = x.shape
        C, L, npre = self.embed_dim, len(layers), self.num_prefix_tokens
        f32 = dict(device=x.device, dtype=torch.float32)
        if concat:
            maps = torch.empty(B, h, w, L * C, **f32)
            dst, ldo = [maps[..., l * C:] for l in range(L)], L * C
        else:
            maps = [torch.empty((B, npre + h * w, C) if all_tokens else (B, h, w, C), **f32) for _ in range(L)]
            dst, ldo = maps, C
        pre = torch.empty(L, B, npre, C, **f32) if prefix else None
        pre_ptrs = (c_void_p * L)(*[pre[l].data_ptr() for l in range(L)]) if prefix else None
        check(lib().dvt_vit_forward_layers(self._handle, ptr(x), 0 if x.dtype == torch.bfloat16 else 1, B, H, W, stride,
                                           ptr(pos_patch), ptr(prefix_rows), ptr(rope), L, (c_int * L)(*layers), int(norm),
                                           (c_void_p * L)(*[t.data_ptr() for t in dst]), ldo, int(all_tokens), pre_ptrs,
                                           cur_stream()), "dvt_vit_forward_layers")
        return maps, pre

    @torch.no_grad()
    def forward_layers_concat(self, x: torch.Tensor, layers: List[int], *, norm: bool, return_cls: bool = False):
        """The maps of `layers` (negative indices count from the end) side by side in channels, in the order given: NHWC
        [B, h, w, len(layers) * C], the `resize_concat` input of the linear probes, from one pass of the blocks.  With
        return_cls also prefix token 0 of each layer, [B, len(layers) * C].  Each map has the bits of
        `get_intermediate_layers` for its layer."""
        depth = len(self.blocks)
        layers = [i if i >= 0 else depth + i for i in layers]
        uniq = sorted(set(layers))
        maps, pre = self._run_layers(x, uniq, norm, concat=True, prefix=return_cls)
        if layers != uniq:  # another order or repeated layers: pick the channel blocks
            pick = torch.tensor([uniq.index(i) for i in layers], device=maps.device)
            B, h, w, _ = maps.shape
            maps = maps.view(B, h, w, len(uniq), -1).index_select(3, pick).reshape(B, h, w, -1)
            pre = pre.index_select(0, pick) if return_cls else None
        if not return_cls:
            return maps
        return maps, pre[:, :, 0].transpose(0, 1).reshape(maps.shape[0], -1)

    def forward_intermediates(self, x, indices=None, return_prefix_tokens=False, norm=False, stop_early=False,
                              output_fmt="NCHW", intermediates_only=False):
        assert output_fmt in ("NCHW", "NLC")
        assert intermediates_only, "only intermediates_only=True is used by DVT (vit_wrapper.py:142)"
        depth = len(self.blocks)
        if indices is None:
            take = list(range(depth))
        elif isinstance(indices, int):
            take = list(range(depth - indices, depth))
        else:
            take = [i if i >= 0 else depth + i for i in indices]
        if self._training():
            # what distillation asks for (reference main_distillation.py:236): one layer, patch tokens only
            if len(take) != 1 or return_prefix_tokens:
                raise NotImplementedError("the ViT training path returns one layer without prefix tokens")
            t = self._run_train(x, take[0], norm)  # [B, h, w, C]
            return [t.permute(0, 3, 1, 2) if output_fmt == "NCHW" else t.reshape(t.shape[0], -1, t.shape[-1])]
        with torch.no_grad():
            return self._forward_intermediates_infer(x, take, return_prefix_tokens, norm, output_fmt)

    def _forward_intermediates_infer(self, x, take, return_prefix_tokens, norm, output_fmt):
        if not take:
            return []
        uniq = sorted(set(take))  # one pass over the blocks serves every requested layer
        maps, _ = self._run_layers(x, uniq, norm, all_tokens=return_prefix_tokens)
        of = dict(zip(uniq, maps))
        outs, seen = [], set()
        for idx in take:
            t = of[idx] if idx not in seen else of[idx].clone()  # a repeated layer gets a tensor of its own
            seen.add(idx)
            if return_prefix_tokens:
                prefix, feat = t[:, :self.num_prefix_tokens], t[:, self.num_prefix_tokens:]
                if output_fmt == "NCHW":
                    H, W = self.patch_embed.dynamic_feat_size((x.shape[2], x.shape[3]))
                    feat = feat.reshape(x.shape[0], H, W, -1).permute(0, 3, 1, 2)
                outs.append((feat, prefix))
            else:  # [B, h, w, C]
                outs.append(t.permute(0, 3, 1, 2) if output_fmt == "NCHW" else t.reshape(t.shape[0], -1, t.shape[-1]))
        return outs

    @torch.no_grad()
    def forward(self, x):
        """num_classes=0 head: pooled (cls) feature after the final norm, as timm's forward_head(pre_logits)."""
        t = self._run(x, len(self.blocks) - 1, True, all_tokens=True)
        return t[:, 0]


class PretrainedViTWrapper(nn.Module):
    def __init__(self, model_identifier: str = "vit_base_patch14_dinov2.lvd142m", stride: int = 7,
                 dynamic_img_size: bool = True, dynamic_img_pad: bool = False, **kwargs):
        super().__init__()
        assert model_identifier in MODEL_LIST, f"Model type {model_identifier} not tested yet."
        self.model_identifier = model_identifier
        self.stride = stride
        self.patch_size = int(re.search(r"patch(\d+)", model_identifier).group(1))
        self.dynamic_img_size = dynamic_img_size
        self.dynamic_img_pad = dynamic_img_pad
        assert dynamic_img_size and not dynamic_img_pad, "the H100 path implements dynamic_img_size=True, no padding"
        self.model, self.transformation = self.create_model(model_identifier, **kwargs)
        # overwrite the stride size (reference vit_wrapper.py:78-79)
        if stride != self.model.patch_embed.proj.stride[0]:
            self.model.patch_embed.proj.stride = [stride, stride]

    @property
    def n_output_dims(self) -> int:
        return self.model.embed_dim

    @property
    def num_blocks(self) -> int:
        return len(self.model.blocks)

    @property
    def last_layer_index(self) -> int:
        return self.num_blocks - 1

    def create_model(self, model_identifier: str, **kwargs):
        from torchvision import transforms
        a = dict(arch_of(model_identifier))
        patch = int(kwargs.pop("patch_size", self.patch_size))
        if "img_size" in kwargs:
            a["img"] = int(kwargs.pop("img_size"))
        # The reference builds the backbone with timm `pretrained=True` and fails hard when the checkpoint cannot be had
        # (vit_wrapper.py:108-112).  Same here: weights come from $DVT_WEIGHTS_DIR/<identifier>.pth; a randomly
        # initialised backbone is an explicit opt-in (tests, bench: `allow_random_init=True` or DVT_ALLOW_RANDOM_INIT=1),
        # never a silent fallback -- stage 1 would otherwise write feature files of a random network that its own resume
        # rule then treats as done.
        allow_random = bool(kwargs.pop("allow_random_init", False)) or os.environ.get("DVT_ALLOW_RANDOM_INIT", "") == "1"
        model = B200VisionTransformer(model_identifier, patch, a)
        wdir = os.environ.get("DVT_WEIGHTS_DIR", "")
        path = os.path.join(wdir, model_identifier + ".pth") if wdir else ""
        self.pretrained_loaded = False
        if path and os.path.isfile(path):
            sd = torch.load(path, map_location="cpu")
            if not is_hf_dinov3_state_dict(sd):   # (HF's DINOv3 layout has `model.layer.*` keys of its own)
                sd = {k[len("model."):] if k.startswith("model.") else k: v for k, v in sd.items()}
            model.load_state_dict(sd, strict=True)
            self.pretrained_loaded = True
        elif allow_random:
            logger.warning("no local weights for %s: random initialisation (explicitly allowed)", model_identifier)
        else:
            raise FileNotFoundError(
                f"pretrained weights for {model_identifier} not found ({path or 'DVT_WEIGHTS_DIR is not set'}); put "
                f"<DVT_WEIGHTS_DIR>/{model_identifier}.pth in place, or pass allow_random_init=True / set "
                "DVT_ALLOW_RANDOM_INIT=1 to run with a randomly initialised backbone")
        size = a["img"]
        transformation = transforms.Compose([
            transforms.Resize(size, interpolation=transforms.InterpolationMode.BICUBIC),
            transforms.CenterCrop(size),
            transforms.ToTensor(),
            transforms.Normalize(mean=a["mean"], std=a["std"]),
        ])
        return model, transformation

    def set_trainable(self, flag: bool = True):
        """Opt in to the training path (stage-3 distillation): with gradients enabled, `get_intermediate_layers` returns a
        differentiable result (one layer, no prefix tokens), for every backbone of `ARCHS`, the SwiGLU ViT-g/14 ones
        included, and of `DINOV3_ARCHS`.  Off by default: the frozen-backbone callers keep the inference forward even when their parameters
        require grad."""
        self.model._trainable = bool(flag)
        return self

    def extract_into(self, x: torch.Tensor, layer_index: int, out_nhwc: torch.Tensor, norm: bool = True) -> torch.Tensor:
        """library-only convenience used by the stage-1 pipeline: writes the [B, h, w, C] map of `layer_index` straight into
        `out_nhwc` (a slice of the feature bank) instead of returning a fresh tensor."""
        return self.model._run(x, layer_index, norm, all_tokens=False, out=out_nhwc)

    def get_intermediate_layers(self, x: torch.Tensor, n: Union[int, List[int], Tuple[int]] = 1, reshape: bool = True,
                                return_prefix_tokens: bool = False, norm: bool = True):
        """Same contract as the reference (vit_wrapper.py:122-143): list of [B, C, H, W] maps (or (map, prefix)
        tuples).  The NCHW tensors are views of the kernel's NHWC output."""
        return self.model.forward_intermediates(x, n, return_prefix_tokens=return_prefix_tokens, norm=norm,
                                                output_fmt="NCHW" if reshape else "NLC", intermediates_only=True)

    def forward(self, x: torch.Tensor):
        return self.model(x)
