"""Stage-2 training operators over torch CUDA tensors (SURVEY.md section 8(f-2)): thin wrappers around the C ABI plus the
two autograd functions the training step is made of -- the denoiser block (`block_forward`) and the distillation loss
(`denoise_loss`).  Every kernel behind them is hand-written sm_90a code of libdvt_b200.so; torch only owns the tensors.

Deterministic training: when `torch.are_deterministic_algorithms_enabled()` is true at call time, the helpers that
reduce with float atomics (`attention_bwd`, `wgrad`, `colsum`, `layernorm_bwd_`, the loss) and the position-embedding
resample (`resample_bicubic`) run fixed-order kernels instead, so that two runs from the same seed on the same GPU model
give bit-identical weights, optimiser moments and losses.  The flag is read at every call.

Reference step (main_denoiser.py:213-220): pred = model(original_feats); loss = mse(pred, denoised) + 1 - mean cosine;
loss.backward(); AdamW.step() -- through timm `Block` (pre-LN attention + GELU MLP, no LayerScale)."""
from __future__ import annotations

import ctypes
from typing import Dict, Tuple

import torch
import torch.nn.functional as F

from . import _lib, ops
from ._lib import DT_BF16, DT_F32, check, cur_stream, lib, ptr


def _dt(t: torch.Tensor) -> int:
    return DT_BF16 if t.dtype == torch.bfloat16 else DT_F32


def _deterministic() -> bool:
    return torch.are_deterministic_algorithms_enabled()


def attention_fwd_lse(qkv: torch.Tensor, heads: int, head_dim: int = 64) -> Tuple[torch.Tensor, torch.Tensor]:
    """qkv bf16 [B, N, 3*heads*head_dim] -> (out bf16 [B, N, heads*head_dim], lse f32 [B, heads, N]); head_dim 64 or 80."""
    assert qkv.is_cuda and qkv.dtype == torch.bfloat16 and qkv.is_contiguous()
    B, N, _ = qkv.shape
    out = torch.empty((B, N, heads * head_dim), device=qkv.device, dtype=torch.bfloat16)
    lse = torch.empty((B, heads, N), device=qkv.device, dtype=torch.float32)
    if head_dim == 64:
        check(lib().dvt_attention_fwd_lse(ptr(qkv), ptr(out), ptr(lse), B, N, heads, cur_stream()), "dvt_attention_fwd_lse")
    else:
        check(lib().dvt_attention_fwd_lse_hd(ptr(qkv), ptr(out), ptr(lse), B, N, heads, head_dim, cur_stream()),
              "dvt_attention_fwd_lse_hd")
    return out, lse


def attention_bwd(qkv: torch.Tensor, out: torch.Tensor, dout: torch.Tensor, lse: torch.Tensor, heads: int,
                  head_dim: int = 64) -> torch.Tensor:
    """Gradient of flash attention w.r.t. qkv (bf16 [B, N, 3C], C = heads * head_dim)."""
    assert all(t.is_cuda and t.is_contiguous() for t in (qkv, out, dout, lse))
    assert qkv.dtype == out.dtype == dout.dtype == torch.bfloat16 and lse.dtype == torch.float32
    B, N, _ = qkv.shape
    dqkv = torch.empty_like(qkv)
    delta = torch.empty((B, heads, N), device=qkv.device, dtype=torch.float32)
    if _deterministic():   # dQ from the query-major kernel, no atomics (dK / dV bits unchanged)
        check(lib().dvt_attention_bwd_det(ptr(qkv), ptr(out), ptr(dout), ptr(lse), ptr(dqkv), ptr(delta), B, N, heads, head_dim,
                                          cur_stream()), "dvt_attention_bwd_det")
        return dqkv
    dq_ws = torch.empty((B, N, heads * head_dim), device=qkv.device, dtype=torch.float32)
    if head_dim == 64:
        check(lib().dvt_attention_bwd(ptr(qkv), ptr(out), ptr(dout), ptr(lse), ptr(dqkv), ptr(dq_ws), ptr(delta), B, N, heads,
                                      cur_stream()), "dvt_attention_bwd")
    else:
        check(lib().dvt_attention_bwd_hd(ptr(qkv), ptr(out), ptr(dout), ptr(lse), ptr(dqkv), ptr(dq_ws), ptr(delta), B, N,
                                         heads, head_dim, cur_stream()), "dvt_attention_bwd_hd")
    return dqkv


def layernorm_bwd_(dx_accum: torch.Tensor, x: torch.Tensor, gamma: torch.Tensor, dy: torch.Tensor, eps: float = 1e-6):
    """dx_accum += dLN/dx; returns (dgamma, dbeta).  x, dy, dx_accum f32 [rows, C] contiguous."""
    if _deterministic():   # the grouped kernel with one row per group is the fixed-order form (same per-row arithmetic)
        return layernorm_bwd_grouped_(dx_accum, x, gamma, dy, 1, 0, eps)
    rows, C = x.shape
    assert all(t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() for t in (dx_accum, x, dy)) and dy.shape == x.shape
    g = gamma.detach().float().contiguous()
    dgamma = torch.zeros(C, device=x.device, dtype=torch.float32)
    dbeta = torch.zeros(C, device=x.device, dtype=torch.float32)
    check(lib().dvt_layernorm_bwd(ptr(x), ptr(g), ptr(dy), ptr(dx_accum), ptr(dgamma), ptr(dbeta), rows, C, eps, cur_stream()),
          "dvt_layernorm_bwd")
    return dgamma, dbeta


def colsum(t: torch.Tensor) -> torch.Tensor:
    """Column sums of a [rows, cols] bf16 / f32 matrix as f32 [cols] (bias gradients)."""
    assert t.is_cuda and t.dim() == 2 and t.stride(1) == 1
    if _deterministic():
        out = torch.empty(t.shape[1], device=t.device, dtype=torch.float32)
        check(lib().dvt_colsum_ordered(ptr(t), _dt(t), t.stride(0), t.shape[0], t.shape[1], ptr(out),
                                       ptr(_workspace(t.shape[1], t.device)), cur_stream()), "dvt_colsum_ordered")
        return out
    out = torch.zeros(t.shape[1], device=t.device, dtype=torch.float32)
    check(lib().dvt_colsum(ptr(t), _dt(t), t.stride(0), t.shape[0], t.shape[1], ptr(out), cur_stream()), "dvt_colsum")
    return out


def gelu(x: torch.Tensor) -> torch.Tensor:
    assert x.is_cuda and x.dtype == torch.bfloat16 and x.is_contiguous()
    out = torch.empty_like(x)
    check(lib().dvt_gelu(ptr(x), ptr(out), x.numel(), cur_stream()), "dvt_gelu")
    return out


def swiglu(hpre: torch.Tensor) -> torch.Tensor:
    """hpre bf16 [rows, 2 Hh] = [g | u] (timm SwiGLUPacked chunk order) -> silu(g) * u bf16 [rows, Hh]; the kernel of the
    inference forward, so both produce the same bits."""
    assert hpre.is_cuda and hpre.dtype == torch.bfloat16 and hpre.is_contiguous() and hpre.dim() == 2 and hpre.shape[1] % 2 == 0
    rows, Hh = hpre.shape[0], hpre.shape[1] // 2
    out = torch.empty((rows, Hh), device=hpre.device, dtype=torch.bfloat16)
    check(lib().dvt_swiglu(ptr(hpre), ptr(out), rows, Hh, cur_stream()), "dvt_swiglu")
    return out


def dgrad_swiglu(dy: torch.Tensor, w2: torch.Tensor, hpre: torch.Tensor) -> torch.Tensor:
    """Gradient w.r.t. the fc1 output of a SwiGLU MLP: dh = dy [rows, C] @ w2 [C, Hh] (fc2's nn.Linear storage, read as an
    MN-major operand; a row pitch larger than Hh is allowed), and the SwiGLU backward on hpre [rows, 2 Hh] in the GEMM
    epilogue -> dhpre bf16 [rows, 2 Hh]."""
    assert dy.dtype == w2.dtype == hpre.dtype == torch.bfloat16 and dy.is_contiguous() and hpre.is_contiguous()
    assert w2.stride(1) == 1 and dy.shape[1] == w2.shape[0] and hpre.shape == (dy.shape[0], 2 * w2.shape[1])
    rows, C = dy.shape
    Hh = w2.shape[1]
    out = torch.empty((rows, 2 * Hh), device=dy.device, dtype=torch.bfloat16)
    check(lib().dvt_gemm_bf16_dgrad_swiglu(ptr(dy), C, ptr(w2), w2.stride(0), rows, Hh, C, ptr(hpre), 2 * Hh, ptr(out), 2 * Hh,
                                           cur_stream()), "dvt_gemm_bf16_dgrad_swiglu")
    return out


def _sms() -> int:
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def dgrad(dy: torch.Tensor, w: torch.Tensor, out_dtype: torch.dtype, gelu_preact: torch.Tensor | None = None) -> torch.Tensor:
    """dx [rows, in] = dy [rows, out] @ w [out, in] (the weight is read in its nn.Linear storage as an MN-major operand);
    optionally multiplied by gelu'(gelu_preact) in the epilogue."""
    assert dy.dtype == w.dtype == torch.bfloat16 and dy.is_contiguous() and w.is_contiguous()
    rows, n_out = dy.shape
    n_in = w.shape[1]
    out = torch.empty((rows, n_in), device=dy.device, dtype=out_dtype)
    pre, ldp = (ptr(gelu_preact), gelu_preact.stride(0)) if gelu_preact is not None else (None, 0)
    check(lib().dvt_gemm_bf16_bwd(ptr(dy), n_out, 0, ptr(w), n_in, 1, rows, n_in, n_out, ptr(out), n_in, _dt(out), 1, pre, ldp,
                                  cur_stream()), "dvt_gemm_bf16_bwd(dgrad)")
    return out


def wgrad_splits(rows: int, n_out: int, n_in: int) -> int:
    """Split-K factor of `wgrad`: enough CTAs to fill the GPU, at least 4 k-blocks of 64 rows per split."""
    wide = n_in >= 256 and (n_in % 256 == 0 or n_in > 1024)
    tiles = ((n_out + 127) // 128) * ((n_in + (255 if wide else 127)) // (256 if wide else 128))
    return max(1, min(_sms() // max(tiles, 1), ((rows + 63) // 64) // 4))


def wgrad(dy: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """dW [out, in] f32 = dy [rows, out]^T @ x [rows, in]: both activations are read in place as MN-major operands; the
    reduction over the rows is split across CTAs (f32 atomics) so that the small output fills the GPU.  Deterministic
    mode: each split stores its partial product into its own workspace plane, and the planes are added in split order."""
    assert dy.dtype == x.dtype == torch.bfloat16 and dy.is_contiguous() and x.is_contiguous() and dy.shape[0] == x.shape[0]
    rows, n_out = dy.shape
    n_in = x.shape[1]
    splits = wgrad_splits(rows, n_out, n_in)
    if _deterministic():
        out = torch.empty((n_out, n_in), device=dy.device, dtype=torch.float32)
        ws = torch.empty(splits * n_out * n_in, device=dy.device, dtype=torch.float32) if splits > 1 else None
        check(lib().dvt_gemm_bf16_wgrad_ordered(ptr(dy), n_out, ptr(x), n_in, n_out, n_in, rows, ptr(out), n_in, splits, ptr(ws),
                                                cur_stream()), "dvt_gemm_bf16_wgrad_ordered")
        return out
    out = (torch.zeros if splits > 1 else torch.empty)((n_out, n_in), device=dy.device, dtype=torch.float32)
    check(lib().dvt_gemm_bf16_bwd(ptr(dy), n_out, 1, ptr(x), n_in, 1, n_out, n_in, rows, ptr(out), n_in, DT_F32, splits, None, 0,
                                  cur_stream()), "dvt_gemm_bf16_bwd(wgrad)")
    return out


def adamw_(p: torch.Tensor, g: torch.Tensor, m: torch.Tensor, v: torch.Tensor, *, lr: float, betas, eps: float,
           weight_decay: float, step: int):
    assert all(t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.numel() == p.numel() for t in (p, g, m, v))
    check(lib().dvt_adamw(ptr(p), ptr(g), ptr(m), ptr(v), p.numel(), float(lr), float(betas[0]), float(betas[1]), float(eps),
                          float(weight_decay), int(step), cur_stream()), "dvt_adamw")


# ---------------------------------------------------------------------------------------------------------------------
# the transformer block of the denoiser as ONE autograd node
# ---------------------------------------------------------------------------------------------------------------------
class _BlockFn(torch.autograd.Function):
    """timm `Block(dim, heads, mlp_ratio=4, qkv_bias=True, init_values=None)` forward / backward on the CUDA kernels.
    Activations kept for the backward pass: the two LayerNorm inputs (f32), their bf16 outputs, qkv, the attention output
    and its log-sum-exp, the MLP pre-activation and activation (bf16)."""

    @staticmethod
    def forward(ctx, x0, n1w, n1b, qkvw, qkvb, projw, projb, n2w, n2b, fc1w, fc1b, fc2w, fc2b, heads: int, batch: int):
        if not x0.is_cuda:
            raise _lib.DvtError("dvt_b200 Denoiser needs CUDA tensors (no CPU fallback)")
        M, C = x0.shape
        N = M // batch
        f32 = lambda t: t.detach().float().contiguous()      # noqa: E731
        b16 = lambda t: t.detach().to(torch.bfloat16).contiguous()  # noqa: E731
        wq, wp, w1, w2 = b16(qkvw), b16(projw), b16(fc1w), b16(fc2w)
        x0 = x0.detach().float().contiguous()
        xn1 = ops.layernorm(x0, f32(n1w), f32(n1b), 1e-6, out_dtype=torch.bfloat16)
        qkv = ops.gemm_tn(xn1, wq, f32(qkvb), None, torch.bfloat16)
        att, lse = attention_fwd_lse(qkv.view(batch, N, 3 * C), heads)
        att = att.view(M, C)
        x1 = x0.clone()
        ops.gemm_tn_residual_(x1, att, wp, f32(projb), None)
        xn2 = ops.layernorm(x1, f32(n2w), f32(n2b), 1e-6, out_dtype=torch.bfloat16)
        hpre = ops.gemm_tn(xn2, w1, f32(fc1b), None, torch.bfloat16)
        hid = gelu(hpre)
        x2 = x1.clone()
        ops.gemm_tn_residual_(x2, hid, w2, f32(fc2b), None)
        ctx.save_for_backward(x0, x1, xn1, qkv, att, lse, xn2, hpre, hid, wq, wp, w1, w2, f32(n1w), f32(n2w))
        ctx.heads, ctx.batch = heads, batch
        return x2

    @staticmethod
    def backward(ctx, dx2):
        x0, x1, xn1, qkv, att, lse, xn2, hpre, hid, wq, wp, w1, w2, n1w, n2w = ctx.saved_tensors
        heads, batch = ctx.heads, ctx.batch
        M, C = x0.shape
        N = M // batch
        dx2 = dx2.detach().float().contiguous()
        d2 = dx2.to(torch.bfloat16)
        # ---- MLP ----
        g_fc2w = wgrad(d2, hid)
        g_fc2b = colsum(dx2)
        dhpre = dgrad(d2, w2, torch.bfloat16, gelu_preact=hpre)
        g_fc1w = wgrad(dhpre, xn2)
        g_fc1b = colsum(dhpre)
        dxn2 = dgrad(dhpre, w1, torch.float32)
        dx1 = dx2.clone()
        g_n2w, g_n2b = layernorm_bwd_(dx1, x1, n2w, dxn2)
        # ---- attention ----
        d1 = dx1.to(torch.bfloat16)
        g_projw = wgrad(d1, att)
        g_projb = colsum(dx1)
        datt = dgrad(d1, wp, torch.bfloat16)
        dqkv = attention_bwd(qkv.view(batch, N, 3 * C), att.view(batch, N, C), datt.view(batch, N, C), lse, heads).view(M, 3 * C)
        g_qkvw = wgrad(dqkv, xn1)
        g_qkvb = colsum(dqkv)
        dxn1 = dgrad(dqkv, wq, torch.float32)
        dx0 = dx1                                     # (dx1 is not needed any more: accumulate in place)
        g_n1w, g_n1b = layernorm_bwd_(dx0, x0, n1w, dxn1)
        return (dx0, g_n1w, g_n1b, g_qkvw, g_qkvb, g_projw, g_projb, g_n2w, g_n2b, g_fc1w, g_fc1b, g_fc2w, g_fc2b, None, None)


def block_forward(x: torch.Tensor, blk, heads: int, batch: int) -> torch.Tensor:
    """x f32 [batch * tokens, C] through one denoiser block (`blk`: module with timm Block parameter names)."""
    return _BlockFn.apply(x, blk.norm1.weight, blk.norm1.bias, blk.attn.qkv.weight, blk.attn.qkv.bias, blk.attn.proj.weight,
                          blk.attn.proj.bias, blk.norm2.weight, blk.norm2.bias, blk.mlp.fc1.weight, blk.mlp.fc1.bias,
                          blk.mlp.fc2.weight, blk.mlp.fc2.bias, heads, batch)


# ---------------------------------------------------------------------------------------------------------------------
# loss
# ---------------------------------------------------------------------------------------------------------------------
class _LossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, pred, target):
        if not pred.is_cuda:
            raise _lib.DvtError("dvt_b200 loss needs CUDA tensors (no CPU fallback)")
        C = pred.shape[-1]
        p = pred.detach().float().contiguous().view(-1, C)
        t = target.detach().float().contiguous().view(-1, C)
        dpred = torch.empty_like(p)
        losses = torch.empty(3, device=p.device, dtype=torch.float32)
        rows = p.shape[0]
        if _deterministic():   # per-CTA partials added in CTA order
            ws = torch.empty(2 * ((rows + 7) // 8), device=p.device, dtype=torch.float32)
            check(lib().dvt_denoise_loss_ordered(ptr(p), ptr(t), ptr(dpred), ptr(losses), ptr(ws), rows, C, 1.0, cur_stream()),
                  "dvt_denoise_loss_ordered")
        else:
            check(lib().dvt_denoise_loss(ptr(p), ptr(t), ptr(dpred), ptr(losses), rows, C, 1.0, cur_stream()), "dvt_denoise_loss")
        ctx.save_for_backward(dpred)
        ctx.shape = pred.shape
        return losses[0], losses[1], losses[2]

    @staticmethod
    def backward(ctx, g_total, g_l2, g_cos):
        (dpred,) = ctx.saved_tensors
        # the step back-propagates `loss` = l2 + cos only (main_denoiser.py:217-219); the two terms are reported values
        return (dpred * g_total).view(ctx.shape), None


def denoise_loss(pred: torch.Tensor, target: torch.Tensor):
    """(loss, l2_loss, cosine_similarity_loss) of main_denoiser.py:214-217 in one kernel; differentiable w.r.t. pred."""
    return _LossFn.apply(pred, target)


# ---------------------------------------------------------------------------------------------------------------------
# position-embedding resampling (timm resample_abs_pos_embed: bicubic, antialias, fp32)
# ---------------------------------------------------------------------------------------------------------------------
_RESAMPLE_W: Dict[tuple, torch.Tensor] = {}


def resample_weights(n_in: int, n_out: int, device) -> torch.Tensor:
    """fp32 [n_out, n_in] weights of F.interpolate(bicubic, antialias=True) along one axis (the op is separable with the same
    1-D weights on both axes), read off ATen itself: a one-hot basis [n_in, 1, n_in] interpolated along its width, the
    height at size 1 -> 1 (the identity).  (A basis along the height with the width at 1 -> 1 does not reproduce the 2-D
    op.)  Cached per shape and device."""
    key = (n_in, n_out, str(device))
    w = _RESAMPLE_W.get(key)
    if w is None:
        with torch.no_grad():
            eye = torch.eye(n_in, device=device, dtype=torch.float32).reshape(1, n_in, 1, n_in)
            w = F.interpolate(eye, size=(1, n_out), mode="bicubic", antialias=True)[0, :, 0, :].t().contiguous()
        _RESAMPLE_W[key] = w
    return w


class _ResampleFn(torch.autograd.Function):
    """F.interpolate(g, (h, w), bicubic, antialias) with a fixed-order backward: the forward is torch's (same bits), the
    backward contracts dout with the exact weight matrices of both axes on the CUDA kernel of dvt_resample_bwd."""

    @staticmethod
    def forward(ctx, g, h: int, w: int):
        ctx.meta = (tuple(g.shape), h, w)
        return F.interpolate(g, size=(h, w), mode="bicubic", antialias=True)

    @staticmethod
    def backward(ctx, dout):
        (_, C, gh, gw), h, w = ctx.meta
        if not dout.is_cuda:
            raise _lib.DvtError("dvt_b200 resample backward needs CUDA tensors (no CPU fallback)")
        dev = dout.device
        wh, ww = resample_weights(gh, h, dev), resample_weights(gw, w, dev)
        d = dout.detach().float()[0].permute(1, 2, 0).contiguous()          # [h, w, C]
        tmp = torch.empty((gh, w, C), device=dev, dtype=torch.float32)
        dgrid = torch.empty((gh, gw, C), device=dev, dtype=torch.float32)
        check(lib().dvt_resample_bwd(ptr(wh), ptr(ww), ptr(d), ptr(tmp), ptr(dgrid), h, w, gh, gw, C, cur_stream()),
              "dvt_resample_bwd")
        return dgrid.permute(2, 0, 1).unsqueeze(0), None, None


def resample_bicubic(g: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """g [1, C, gh, gw] fp32 -> F.interpolate(g, (h, w), bicubic, antialias=True), differentiable; in deterministic mode the
    backward is the fixed-order kernel (torch's CUDA backward of this op adds with atomics)."""
    if _deterministic():
        return _ResampleFn.apply(g, h, w)
    return F.interpolate(g, size=(h, w), mode="bicubic", antialias=True)


# ---------------------------------------------------------------------------------------------------------------------
# stage 3 (distillation, reference main_distillation.py): the whole ViT backbone as autograd nodes -- token assembly,
# pre-LN blocks with optional LayerScale, final LayerNorm with the prefix strip
# ---------------------------------------------------------------------------------------------------------------------
_WS_ROWS = 256     # workspace rows (of C floats) of the fixed-order column sums (include/dvt_b200.h, stage 3)


def _workspace(C: int, device) -> torch.Tensor:
    return torch.empty(_WS_ROWS * C, device=device, dtype=torch.float32)


def gemm_tn_residual_ex_(x: torch.Tensor, a: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None,
                         gamma: torch.Tensor | None, branch: torch.Tensor | None) -> torch.Tensor:
    """x += gamma * (a @ w.T + bias) in place (fp32 x); when `branch` (bf16 [M, N]) is given, it receives a @ w.T + bias."""
    assert x.is_cuda and x.dtype == torch.float32 and x.stride(1) == 1
    M, K = a.shape
    N = w.shape[0]
    if branch is not None:
        assert branch.dtype == torch.bfloat16 and branch.shape == (M, N) and branch.is_contiguous()
    check(lib().dvt_gemm_tn_residual_ex(ptr(a), a.stride(0), ptr(w), w.stride(0), _dt(a), M, N, K, ptr(bias), ptr(gamma), ptr(x),
                                        x.stride(0), ptr(branch), N, cur_stream()), "dvt_gemm_tn_residual_ex")
    return x


def layerscale_bwd(dx: torch.Tensor, branch: torch.Tensor | None, gamma: torch.Tensor | None, want_dbranch: bool = True):
    """Backward of x += gamma * branch: (dbranch bf16 = gamma * dx, dbias = sum_rows gamma * dx, dgamma = sum_rows dx *
    branch or None).  gamma None: no LayerScale (cast + column sum).  Fixed-order sums: bit-identical across calls."""
    assert dx.is_cuda and dx.dtype == torch.float32 and dx.dim() == 2 and dx.stride(1) == 1
    rows, C = dx.shape
    dbranch = torch.empty((rows, C), device=dx.device, dtype=torch.bfloat16) if want_dbranch else None
    dbias = torch.empty(C, device=dx.device, dtype=torch.float32)
    dgamma = None
    if gamma is not None:
        gamma = gamma.detach().float().contiguous()
        if branch is not None:
            assert branch.dtype == torch.bfloat16 and branch.shape == (rows, C) and branch.is_contiguous()
            dgamma = torch.empty(C, device=dx.device, dtype=torch.float32)
    check(lib().dvt_layerscale_bwd(ptr(dx), dx.stride(0), ptr(branch if dgamma is not None else None), ptr(gamma), ptr(dbranch),
                                   ptr(dbias), ptr(dgamma), ptr(_workspace(C, dx.device)), rows, C, cur_stream()),
          "dvt_layerscale_bwd")
    return dbranch, dbias, dgamma


def vit_embed_bwd(dx0: torch.Tensor, batch: int, prefix: int):
    """dx0 f32 [batch * ntok, C] -> (dpatch bf16 [batch * np, C], dpos f32 [np, C], dprefix f32 [prefix, C], dbias f32 [C])."""
    assert dx0.is_cuda and dx0.dtype == torch.float32 and dx0.is_contiguous()
    M, C = dx0.shape
    ntok = M // batch
    np_ = ntok - prefix
    dev = dx0.device
    dpatch = torch.empty((batch * np_, C), device=dev, dtype=torch.bfloat16)
    dpos = torch.empty((np_, C), device=dev, dtype=torch.float32)
    dprefix = torch.empty((prefix, C), device=dev, dtype=torch.float32)
    dbias = torch.empty(C, device=dev, dtype=torch.float32)
    check(lib().dvt_vit_embed_bwd(ptr(dx0), batch, ntok, prefix, C, ptr(dpatch), ptr(dpos), ptr(dprefix), ptr(dbias),
                                  ptr(_workspace(C, dev)), cur_stream()), "dvt_vit_embed_bwd")
    return dpatch, dpos, dprefix, dbias


def layernorm_bwd_grouped_(dx_accum: torch.Tensor, x: torch.Tensor, gamma: torch.Tensor, dy: torch.Tensor, in_group: int,
                           skip: int, eps: float = 1e-6):
    """Backward of ops.layernorm(x, ..., in_group, skip): dy holds the compacted rows; dx_accum += dLN/dx on the kept rows
    of the full [rows, C] tensor; returns (dgamma, dbeta) (fixed-order sums)."""
    rows, C = x.shape
    assert all(t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() for t in (dx_accum, x, dy))
    assert dx_accum.shape == x.shape and dy.shape == (rows // in_group * (in_group - skip), C)
    g = gamma.detach().float().contiguous()
    dgamma = torch.empty(C, device=x.device, dtype=torch.float32)
    dbeta = torch.empty(C, device=x.device, dtype=torch.float32)
    check(lib().dvt_layernorm_bwd_grouped(ptr(x), ptr(g), ptr(dy), ptr(dx_accum), ptr(dgamma), ptr(dbeta),
                                          ptr(_workspace(C, x.device)), rows, C, eps, in_group, skip, cur_stream()),
          "dvt_layernorm_bwd_grouped")
    return dgamma, dbeta


class _VitEmbedFn(torch.autograd.Function):
    """Patch embedding (im2col -> GEMM + bias + position) and the prefix rows, as in dvt_vit_forward.  The image gets no
    gradient; pos_patch [np, C] and prefix_rows [prefix, C] are tensors of the caller's graph (built from pos_embed /
    cls_token / reg_token), so autograd carries their gradients on to the parameters."""

    @staticmethod
    def forward(ctx, img, pe_w, pe_b, pos_patch, prefix_rows, stride: int):
        if not img.is_cuda:
            raise _lib.DvtError("dvt_b200 ViT training needs CUDA tensors (no CPU fallback)")
        C, _, P, _ = pe_w.shape
        K = 3 * P * P
        Kp = (K + 7) // 8 * 8
        B, _, H, W = img.shape
        h, w = (H - P) // stride + 1, (W - P) // stride + 1
        np_, prefix = h * w, prefix_rows.shape[0]
        patches = ops.im2col(img.detach().contiguous(), P, stride)
        wpad = torch.nn.functional.pad(pe_w.detach().float().reshape(C, K), (0, Kp - K)).to(torch.bfloat16).contiguous()
        out = torch.empty((B * (np_ + prefix), C), device=img.device, dtype=torch.float32)
        pp = pos_patch.detach().float().contiguous()
        pr = prefix_rows.detach().float().contiguous()
        bias = None if pe_b is None else pe_b.detach().float().contiguous()   # None: patch embedding without bias (CLIP)
        check(lib().dvt_vit_embed_fwd(ptr(patches), Kp, ptr(wpad), ptr(bias), ptr(pp), ptr(pr), B, np_, prefix, C, ptr(out),
                                      cur_stream()), "dvt_vit_embed_fwd")
        ctx.save_for_backward(patches)
        ctx.meta = (B, prefix, C, P, K)
        ctx.has_bias = pe_b is not None
        return out

    @staticmethod
    def backward(ctx, dx0):
        (patches,) = ctx.saved_tensors
        B, prefix, C, P, K = ctx.meta
        dpatch, dpos, dprefix, dbias = vit_embed_bwd(dx0.detach().float().contiguous(), B, prefix)
        gw = wgrad(dpatch, patches)[:, :K].reshape(C, 3, P, P)
        return None, gw, (dbias if ctx.has_bias else None), dpos, dprefix, None


def vit_embed(img: torch.Tensor, patch_embed_w, patch_embed_b, pos_patch, prefix_rows, stride: int) -> torch.Tensor:
    """Token rows f32 [B * (prefix + h*w), C] of images [B, 3, H, W] (f32 or bf16).  patch_embed_b None: no bias (and no
    bias gradient)."""
    return _VitEmbedFn.apply(img, patch_embed_w, patch_embed_b, pos_patch, prefix_rows, stride)


class _VitLayerNormFn(torch.autograd.Function):
    """LayerNorm over every token row, f32 in and out (timm `norm_pre` of the pre_norm ViTs, the CLIP towers); backward
    through dvt_layernorm_bwd."""

    @staticmethod
    def forward(ctx, x, w, b, eps: float):
        if not x.is_cuda:
            raise _lib.DvtError("dvt_b200 ViT training needs CUDA tensors (no CPU fallback)")
        x = x.detach().float().contiguous()
        wf, bf = w.detach().float().contiguous(), b.detach().float().contiguous()
        y = ops.layernorm(x, wf, bf, eps, out_dtype=torch.float32)
        ctx.save_for_backward(x, wf)
        ctx.eps = eps
        return y

    @staticmethod
    def backward(ctx, dy):
        x, wf = ctx.saved_tensors
        dx = torch.zeros_like(x)
        dg, db = layernorm_bwd_(dx, x, wf, dy.detach().float().contiguous(), ctx.eps)
        return dx, dg, db, None


def vit_layernorm(x: torch.Tensor, w, b, eps: float = 1e-6) -> torch.Tensor:
    """x f32 [rows, C] -> LayerNorm(x) f32 [rows, C], differentiable w.r.t. x, w and b."""
    return _VitLayerNormFn.apply(x, w, b, eps)


def _is_swiglu(w1: torch.Tensor, w2: torch.Tensor) -> bool:
    """SwiGLUPacked MLP (ViT-g/14): fc2's input width is half of fc1's output width."""
    return 2 * w2.shape[1] == w1.shape[0]


def _vit_block_fwd(x0, wts, heads: int, batch: int, keep: bool, eps: float = 1e-6):
    """Forward of one pre-LN ViT block on prepared weights; returns (x2, activations for the backward or None).  The MLP is
    GELU, or SwiGLU when fc2's input width is half of fc1's output width."""
    n1w, n1b, wq, qkvb, wp, projb, ls1, n2w, n2b, w1, fc1b, w2, fc2b, ls2 = wts
    M, C = x0.shape
    N = M // batch
    xn1 = ops.layernorm(x0, n1w, n1b, eps, out_dtype=torch.bfloat16)
    qkv = ops.gemm_tn(xn1, wq, qkvb, None, torch.bfloat16)
    att, lse = attention_fwd_lse(qkv.view(batch, N, 3 * C), heads, C // heads)
    att = att.view(M, C)
    branch = lambda g: torch.empty((M, C), device=x0.device, dtype=torch.bfloat16) if (keep and g is not None) else None  # noqa
    x1 = x0.clone()
    br1 = branch(ls1)
    gemm_tn_residual_ex_(x1, att, wp, projb, ls1, br1)
    xn2 = ops.layernorm(x1, n2w, n2b, eps, out_dtype=torch.bfloat16)
    hpre = ops.gemm_tn(xn2, w1, fc1b, None, torch.bfloat16)
    hid = swiglu(hpre) if _is_swiglu(w1, w2) else gelu(hpre)
    x2 = x1.clone()
    br2 = branch(ls2)
    gemm_tn_residual_ex_(x2, hid, w2, fc2b, ls2, br2)
    return x2, ((x1, xn1, qkv, att, lse, br1, xn2, hpre, hid, br2) if keep else None)


class _VitBlockFn(torch.autograd.Function):
    """timm ViT `Block` (pre-LN attention + GELU or SwiGLUPacked MLP, LayerScale ls1 / ls2 when given) forward / backward on
    the CUDA kernels; bf16 GEMM operands, fp32 residual stream and fp32 master weights, as `_BlockFn`.  Saved for the
    backward: what `_BlockFn` saves, plus the bf16 pre-LayerScale branch values of the two residual GEMMs (LayerScale blocks
    only); for SwiGLU the MLP pair is the fc1 output [g | u] (bf16 [M, 2 Hh]) and silu(g) * u (bf16 [M, Hh]).
    checkpoint=True saves the block input only and recomputes the forward during the backward."""

    @staticmethod
    def forward(ctx, x0, n1w, n1b, qkvw, qkvb, projw, projb, ls1, n2w, n2b, fc1w, fc1b, fc2w, fc2b, ls2, heads: int, batch: int,
                checkpoint: bool, eps: float):
        if not x0.is_cuda:
            raise _lib.DvtError("dvt_b200 ViT training needs CUDA tensors (no CPU fallback)")
        f32 = lambda t: None if t is None else t.detach().float().contiguous()      # noqa: E731
        b16 = lambda t: t.detach().to(torch.bfloat16).contiguous()                   # noqa: E731
        wts = (f32(n1w), f32(n1b), b16(qkvw), f32(qkvb), b16(projw), f32(projb), f32(ls1), f32(n2w), f32(n2b), b16(fc1w),
               f32(fc1b), b16(fc2w), f32(fc2b), f32(ls2))
        x0 = x0.detach().float().contiguous()
        x2, acts = _vit_block_fwd(x0, wts, heads, batch, keep=not checkpoint, eps=eps)
        ctx.wts, ctx.heads, ctx.batch, ctx.checkpoint, ctx.eps = wts, heads, batch, checkpoint, eps
        ctx.save_for_backward(x0, *(acts if acts is not None else ()))
        return x2

    @staticmethod
    def backward(ctx, dx2):
        x0, *acts = ctx.saved_tensors
        wts, heads, batch, eps = ctx.wts, ctx.heads, ctx.batch, ctx.eps
        n1w, _, wq, _, wp, _, ls1, n2w, _, w1, _, w2, _, ls2 = wts
        if ctx.checkpoint:
            _, acts = _vit_block_fwd(x0, wts, heads, batch, keep=True, eps=eps)
        x1, xn1, qkv, att, lse, br1, xn2, hpre, hid, br2 = acts
        M, C = x0.shape
        N = M // batch
        dx2 = dx2.detach().float().contiguous()
        # ---- MLP branch: x2 = x1 + ls2 * fc2(act(fc1(LN2(x1)))), act = gelu or swiglu ----
        d2, g_fc2b, g_ls2 = layerscale_bwd(dx2, br2, ls2)
        g_fc2w = wgrad(d2, hid)
        if _is_swiglu(w1, w2):
            dhpre = dgrad_swiglu(d2, w2, hpre)
        else:
            dhpre = dgrad(d2, w2, torch.bfloat16, gelu_preact=hpre)
        g_fc1w = wgrad(dhpre, xn2)
        g_fc1b = colsum(dhpre)
        dxn2 = dgrad(dhpre, w1, torch.float32)
        dx1 = dx2.clone()
        g_n2w, g_n2b = layernorm_bwd_(dx1, x1, n2w, dxn2, eps)
        # ---- attention branch: x1 = x0 + ls1 * proj(attn(qkv(LN1(x0)))) ----
        d1, g_projb, g_ls1 = layerscale_bwd(dx1, br1, ls1)
        g_projw = wgrad(d1, att)
        datt = dgrad(d1, wp, torch.bfloat16)
        dqkv = attention_bwd(qkv.view(batch, N, 3 * C), att.view(batch, N, C), datt.view(batch, N, C), lse, heads,
                             C // heads).view(M, 3 * C)
        g_qkvw = wgrad(dqkv, xn1)
        g_qkvb = colsum(dqkv)
        dxn1 = dgrad(dqkv, wq, torch.float32)
        dx0 = dx1
        g_n1w, g_n1b = layernorm_bwd_(dx0, x0, n1w, dxn1, eps)
        return (dx0, g_n1w, g_n1b, g_qkvw, g_qkvb, g_projw, g_projb, g_ls1, g_n2w, g_n2b, g_fc1w, g_fc1b, g_fc2w, g_fc2b, g_ls2,
                None, None, None, None)


def vit_block_forward(x: torch.Tensor, blk, heads: int, batch: int, checkpoint: bool = False,
                      eps: float = 1e-6) -> torch.Tensor:
    """x f32 [batch * tokens, C] through one ViT block (`blk`: module with timm Block parameter names; ls1 / ls2 either
    LayerScale modules with `gamma` or identities).  head_dim = C / heads (64 or 80); eps of both LayerNorms."""
    ls1 = getattr(blk.ls1, "gamma", None)
    ls2 = getattr(blk.ls2, "gamma", None)
    return _VitBlockFn.apply(x, blk.norm1.weight, blk.norm1.bias, blk.attn.qkv.weight, blk.attn.qkv.bias, blk.attn.proj.weight,
                             blk.attn.proj.bias, ls1, blk.norm2.weight, blk.norm2.bias, blk.mlp.fc1.weight, blk.mlp.fc1.bias,
                             blk.mlp.fc2.weight, blk.mlp.fc2.bias, ls2, heads, batch, checkpoint, eps)


class _VitNormStripFn(torch.autograd.Function):
    """Final LayerNorm over the token rows with the prefix tokens dropped (dvt_layernorm in_group / skip form): x f32
    [B * ntok, C] -> f32 [B * (ntok - prefix), C]; backward through dvt_layernorm_bwd_grouped (prefix rows get zero)."""

    @staticmethod
    def forward(ctx, x, w, b, ntok: int, prefix: int, eps: float):
        x = x.detach().float().contiguous()
        wf, bf = w.detach().float().contiguous(), b.detach().float().contiguous()
        y = ops.layernorm(x, wf, bf, eps, out_dtype=torch.float32, in_group=ntok, skip=prefix)
        ctx.save_for_backward(x, wf)
        ctx.meta = (ntok, prefix, eps)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, wf = ctx.saved_tensors
        ntok, prefix, eps = ctx.meta
        dx = torch.zeros_like(x)
        dg, db = layernorm_bwd_grouped_(dx, x, wf, dy.detach().float().contiguous(), ntok, prefix, eps)
        return dx, dg, db, None, None, None


def vit_norm_strip(x: torch.Tensor, w, b, ntok: int, prefix: int, eps: float = 1e-6) -> torch.Tensor:
    return _VitNormStripFn.apply(x, w, b, ntok, prefix, eps)
