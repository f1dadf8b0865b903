"""Stage-2 training operators over torch CUDA tensors (SURVEY.md section 8(f-2)): thin wrappers around the C ABI plus the
two autograd functions the training step is made of -- the denoiser block (`block_forward`) and the distillation loss
(`denoise_loss`).  Every kernel behind them is hand-written sm_90a code of libdvt_b200.so; torch only owns the tensors.

Reference step (main_denoiser.py:213-220): pred = model(original_feats); loss = mse(pred, denoised) + 1 - mean cosine;
loss.backward(); AdamW.step() -- through timm `Block` (pre-LN attention + GELU MLP, no LayerScale)."""
from __future__ import annotations

import ctypes
from typing import Tuple

import torch

from . import _lib, ops
from ._lib import DT_BF16, DT_F32, check, cur_stream, lib, ptr


def _dt(t: torch.Tensor) -> int:
    return DT_BF16 if t.dtype == torch.bfloat16 else DT_F32


def attention_fwd_lse(qkv: torch.Tensor, heads: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """qkv bf16 [B, N, 3*heads*64] -> (out bf16 [B, N, heads*64], lse f32 [B, heads, N])."""
    assert qkv.is_cuda and qkv.dtype == torch.bfloat16 and qkv.is_contiguous()
    B, N, _ = qkv.shape
    out = torch.empty((B, N, heads * 64), device=qkv.device, dtype=torch.bfloat16)
    lse = torch.empty((B, heads, N), device=qkv.device, dtype=torch.float32)
    check(lib().dvt_attention_fwd_lse(ptr(qkv), ptr(out), ptr(lse), B, N, heads, cur_stream()), "dvt_attention_fwd_lse")
    return out, lse


def attention_bwd(qkv: torch.Tensor, out: torch.Tensor, dout: torch.Tensor, lse: torch.Tensor, heads: int) -> torch.Tensor:
    """Gradient of flash attention w.r.t. qkv (bf16 [B, N, 3C])."""
    assert all(t.is_cuda and t.is_contiguous() for t in (qkv, out, dout, lse))
    assert qkv.dtype == out.dtype == dout.dtype == torch.bfloat16 and lse.dtype == torch.float32
    B, N, _ = qkv.shape
    dqkv = torch.empty_like(qkv)
    dq_ws = torch.empty((B, N, heads * 64), device=qkv.device, dtype=torch.float32)
    delta = torch.empty((B, heads, N), device=qkv.device, dtype=torch.float32)
    check(lib().dvt_attention_bwd(ptr(qkv), ptr(out), ptr(dout), ptr(lse), ptr(dqkv), ptr(dq_ws), ptr(delta), B, N, heads,
                                  cur_stream()), "dvt_attention_bwd")
    return dqkv


def layernorm_bwd_(dx_accum: torch.Tensor, x: torch.Tensor, gamma: torch.Tensor, dy: torch.Tensor, eps: float = 1e-6):
    """dx_accum += dLN/dx; returns (dgamma, dbeta).  x, dy, dx_accum f32 [rows, C] contiguous."""
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
    out = torch.zeros(t.shape[1], device=t.device, dtype=torch.float32)
    check(lib().dvt_colsum(ptr(t), _dt(t), t.stride(0), t.shape[0], t.shape[1], ptr(out), cur_stream()), "dvt_colsum")
    return out


def gelu(x: torch.Tensor) -> torch.Tensor:
    assert x.is_cuda and x.dtype == torch.bfloat16 and x.is_contiguous()
    out = torch.empty_like(x)
    check(lib().dvt_gelu(ptr(x), ptr(out), x.numel(), cur_stream()), "dvt_gelu")
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


def wgrad(dy: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """dW [out, in] f32 = dy [rows, out]^T @ x [rows, in]: both activations are read in place as MN-major operands; the
    reduction over the rows is split across CTAs (f32 atomics) so that the small output fills the GPU."""
    assert dy.dtype == x.dtype == torch.bfloat16 and dy.is_contiguous() and x.is_contiguous() and dy.shape[0] == x.shape[0]
    rows, n_out = dy.shape
    n_in = x.shape[1]
    wide = n_in >= 256 and (n_in % 256 == 0 or n_in > 1024)
    tiles = ((n_out + 127) // 128) * ((n_in + (255 if wide else 127)) // (256 if wide else 128))
    splits = max(1, min(_sms() // max(tiles, 1), ((rows + 63) // 64) // 4))
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
        check(lib().dvt_denoise_loss(ptr(p), ptr(t), ptr(dpred), ptr(losses), p.shape[0], C, 1.0, cur_stream()), "dvt_denoise_loss")
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
