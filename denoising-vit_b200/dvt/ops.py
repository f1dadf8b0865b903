"""Unit operators over torch CUDA tensors (thin wrappers around the C ABI; used by tests and by dvt.models)."""
from __future__ import annotations

import ctypes

import torch

from . import _lib
from ._lib import DT_BF16, DT_F32, DvtError, check, cur_stream, lib, ptr  # noqa: F401

_ACT = {None: 0, "none": 0, "gelu": 1, "relu": 2}


def _dt(t: torch.Tensor) -> int:
    if t.dtype == torch.bfloat16:
        return DT_BF16
    if t.dtype == torch.float32:
        return DT_F32
    raise TypeError(f"unsupported dtype {t.dtype}")


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.DvtError("dvt_b200 operators need CUDA tensors (no CPU fallback)")


def gemm_tn(a: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None = None, act: str | None = None,
            out_dtype: torch.dtype = torch.bfloat16, splits: int = 1, out: torch.Tensor | None = None) -> torch.Tensor:
    """out = act(a @ w.T + bias); a [M,K], w [N,K] (nn.Linear weight layout)."""
    _need_cuda(a, w, bias)
    assert a.dim() == 2 and w.dim() == 2 and a.shape[1] == w.shape[1] and a.dtype == w.dtype
    assert a.stride(1) == 1 and w.stride(1) == 1
    M, K = a.shape
    N = w.shape[0]
    if out is None:
        out = (torch.zeros if splits > 1 else torch.empty)((M, N), device=a.device, dtype=out_dtype)
    check(lib().dvt_gemm_tn(ptr(a), a.stride(0), ptr(w), w.stride(0), _dt(a), M, N, K, ptr(bias), _ACT[act], ptr(out),
                            out.stride(0), _dt(out), splits, cur_stream()), "dvt_gemm_tn")
    return out


def gemm_tn_residual_(x: torch.Tensor, a: torch.Tensor, w: torch.Tensor, bias: torch.Tensor | None,
                      gamma: torch.Tensor | None) -> torch.Tensor:
    """x += gamma * (a @ w.T + bias), x fp32 [M,N] in place."""
    _need_cuda(x, a, w, bias, gamma)
    assert x.dtype == torch.float32 and x.stride(1) == 1
    M, K = a.shape
    N = w.shape[0]
    check(lib().dvt_gemm_tn_residual(ptr(a), a.stride(0), ptr(w), w.stride(0), _dt(a), M, N, K, ptr(bias), ptr(gamma),
                                     ptr(x), x.stride(0), cur_stream()), "dvt_gemm_tn_residual")
    return x


def layernorm(x: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, eps: float = 1e-6,
              out_dtype: torch.dtype = torch.bfloat16, in_group: int = 1, skip: int = 0) -> torch.Tensor:
    """Row LayerNorm of fp32 x [rows, C]; optional prefix strip (drop the first `skip` rows of every `in_group`)."""
    _need_cuda(x, gamma, beta)
    assert x.dim() == 2 and x.dtype == torch.float32 and x.stride(1) == 1
    rows, C = x.shape
    out_rows = rows if skip == 0 else rows // in_group * (in_group - skip)
    y = torch.empty((out_rows, C), device=x.device, dtype=out_dtype)
    check(lib().dvt_layernorm(ptr(x), x.stride(0), ptr(gamma), ptr(beta), ptr(y), y.stride(0), _dt(y), rows, C, eps,
                              in_group, skip, cur_stream()), "dvt_layernorm")
    return y


def attention(qkv: torch.Tensor, heads: int, head_dim: int = 64) -> torch.Tensor:
    """qkv bf16 [B, N, 3*heads*head_dim] (timm Attention.qkv output) -> bf16 [B, N, heads*head_dim]; head_dim 64 or 80."""
    _need_cuda(qkv)
    assert qkv.dtype == torch.bfloat16 and qkv.is_contiguous() and qkv.shape[2] == 3 * heads * head_dim
    B, N, _ = qkv.shape
    out = torch.empty((B, N, heads * head_dim), device=qkv.device, dtype=torch.bfloat16)
    if head_dim == 64:
        check(lib().dvt_attention_fwd(ptr(qkv), ptr(out), B, N, heads, cur_stream()), "dvt_attention_fwd")
    else:
        check(lib().dvt_attention_fwd_hd(ptr(qkv), ptr(out), B, N, heads, head_dim, cur_stream()), "dvt_attention_fwd_hd")
    return out


def im2col(x: torch.Tensor, patch: int, stride: int) -> torch.Tensor:
    """x [B,3,H,W] f32/bf16 -> bf16 [B*h*w, round_up(3*P*P, 8)]."""
    _need_cuda(x)
    assert x.dim() == 4 and x.shape[1] == 3 and x.is_contiguous()
    B, _, H, W = x.shape
    h, w = (H - patch) // stride + 1, (W - patch) // stride + 1
    kp = (3 * patch * patch + 7) // 8 * 8
    out = torch.empty((B * h * w, kp), device=x.device, dtype=torch.bfloat16)
    check(lib().dvt_im2col(ptr(x), _dt(x), ptr(out), B, H, W, patch, stride, cur_stream()), "dvt_im2col")
    return out


def gemm_bf16_ex(a: torch.Tensor, b: torch.Tensor, M: int, N: int, K: int, a_mn: bool = False, b_mn: bool = False,
                 out_dtype: torch.dtype = torch.float32, splits: int = 1, last_col: bool = False):
    """out[M,N] = A . B^T with A given as [M,K] (a_mn False) or [K,M] (a_mn True); B as [N,K] or [K,N]."""
    _need_cuda(a, b)
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16 and a.stride(1) == 1 and b.stride(1) == 1
    atomic = splits > 1 or last_col
    n_out = N - 1 if last_col else N
    ldo = (n_out + 3) // 4 * 4
    out = (torch.zeros if atomic else torch.empty)((M, ldo), device=a.device, dtype=out_dtype)
    lc = torch.zeros(M, device=a.device, dtype=torch.float32) if last_col else None
    check(lib().dvt_gemm_bf16_ex(ptr(a), a.stride(0), int(a_mn), ptr(b), b.stride(0), int(b_mn), M, N, K, ptr(out),
                                 out.stride(0), _dt(out), splits, ptr(lc), cur_stream()), "dvt_gemm_bf16_ex")
    return (out[:, :n_out], lc) if last_col else out[:, :n_out]


def split_tf32(x: torch.Tensor) -> torch.Tensor:
    """fp32 [..] -> [2, ..]: plane 0 = TF32-exact part (low 13 mantissa bits cleared), plane 1 = remainder."""
    hi = (x.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)
    return torch.stack([hi, x - hi]).contiguous()


def gemm_f32x3(a: torch.Tensor, b: torch.Tensor, M: int, N: int, K: int, a_mn: bool = False, b_mn: bool = False,
               splits: int = 1, last_col: bool = False):
    """fp32-accurate product of fp32 matrices on the tensor cores (3xTF32).  a / b are plain fp32 matrices
    ([M,K] or [K,M] when a_mn; [N,K] or [K,N] when b_mn); they are split into hi/lo planes here."""
    _need_cuda(a, b)
    ap, bp = split_tf32(a), split_tf32(b)
    atomic = splits > 1 or last_col
    n_out = N - 1 if last_col else N
    ldo = (n_out + 3) // 4 * 4
    out = (torch.zeros if atomic else torch.empty)((M, ldo), device=a.device, dtype=torch.float32)
    lc = torch.zeros(M, device=a.device, dtype=torch.float32) if last_col else None
    check(lib().dvt_gemm_f32x3(ptr(ap), a.shape[1], a.numel(), int(a_mn), ptr(bp), b.shape[1], b.numel(), int(b_mn), M, N,
                               K, ptr(out), out.stride(0), splits, ptr(lc), cur_stream()), "dvt_gemm_f32x3")
    return (out[:, :n_out], lc) if last_col else out[:, :n_out]


def view_crops(image: torch.Tensor, boxes, flips, size, hp: int, wp: int, out: torch.Tensor | None = None,
               coords_out: torch.Tensor | None = None, dtype: torch.dtype = torch.float32):
    """All views of one image in one launch: out[v] = hflip?(resized_crop(image, boxes[v], size, BICUBIC, antialias=True)),
    coords_out[v] = the (x, y) patch-coordinate grid of the crop (reference: dvt/dataset/transform.py:39-76).
    image f32 cuda [3, H, W]; boxes int [V, 4] (top, left, height, width) and flips int [V] on the HOST."""
    import numpy as np
    _need_cuda(image)
    assert image.dtype == torch.float32 and image.is_contiguous() and image.dim() == 3 and image.shape[0] == 3
    b = np.ascontiguousarray(np.asarray(boxes, dtype=np.int32).reshape(-1, 4))
    f = np.ascontiguousarray(np.asarray(flips, dtype=np.int32).reshape(-1))
    V = b.shape[0]
    assert f.shape[0] == V
    OH, OW = int(size[0]), int(size[1])
    if out is None:
        out = torch.empty((V, 3, OH, OW), device=image.device, dtype=dtype)
    if coords_out is None:
        coords_out = torch.empty((V, hp, wp, 2), device=image.device, dtype=torch.float32)
    assert out.is_contiguous() and tuple(out.shape) == (V, 3, OH, OW) and out.dtype in (torch.float32, torch.bfloat16)
    assert coords_out.is_contiguous() and tuple(coords_out.shape) == (V, hp, wp, 2) and coords_out.dtype == torch.float32
    check(lib().dvt_view_crops(ptr(image), image.shape[1], image.shape[2], b.ctypes.data_as(ctypes.c_void_p),
                               f.ctypes.data_as(ctypes.c_void_p), V, ptr(out), _dt(out), OH, OW, ptr(coords_out), hp, wp,
                               cur_stream()), "dvt_view_crops")
    return out, coords_out
