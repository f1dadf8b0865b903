"""torch bindings of the depth-probe kernels (include/dvt_b200.h, `dvt_depth_*`) and the depth losses.

The head's n_bins logits are computed at the feature grid (`head_logits`, a torch GEMM: the 1x1 conv commutes with the
bilinear upsample of the reference and the cls half of the conv is one vector per image); the kernels interpolate them
at the upsampled grid, take the bin expectation, resize to the ground truth and evaluate.  The reference's
full-resolution features and logits never exist."""
from __future__ import annotations

from typing import Sequence

import torch
import torch.nn.functional as F

from .._lib import DvtError, check, cur_stream, lib, ptr

EVAL_WORKSPACE = 1280   # f64 entries: 128 CTAs x 10 partial sums
LOSS_EPS = 1e-3         # SigLoss / GradientLoss eps


def _need_cuda(*ts):
    for t in ts:
        if not t.is_cuda:
            raise DvtError("dvt_b200 depth kernels need CUDA tensors (no CPU fallback)")
        if t.dtype != torch.float32:
            raise DvtError(f"dvt_b200 depth kernels take float32 tensors, got {t.dtype}")


def head_logits(feat: torch.Tensor, cls: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor, n_maps: int = 1):
    """BNHead conv_depth at the feature grid.  feat NHWC [B, h, w, n C] (n maps of C channels), cls [B, n C]; weight
    [K, 2 n C, 1, 1] whose input channels are (map_0, cls_0, map_1, cls_1, ...), the reference's cat((x, cls), 1) per
    map -> logits NHWC [B, h, w, K]."""
    K = weight.shape[0]
    w2 = weight.reshape(K, -1)
    nc = feat.shape[-1]
    if w2.shape[1] != 2 * nc or cls.shape[-1] != nc or nc % n_maps:
        raise DvtError(f"depth head: conv_depth takes {w2.shape[1]} channels; features give {nc} and cls {cls.shape[-1]}")
    C = nc // n_maps
    cols = torch.arange(2 * nc, device=weight.device).view(n_maps, 2, C)
    w_patch, w_cls = w2[:, cols[:, 0].reshape(-1)], w2[:, cols[:, 1].reshape(-1)]
    return F.linear(feat, w_patch) + (F.linear(cls, w_cls) + bias)[:, None, None, :]


def head_depth(logits: torch.Tensor, bins: torch.Tensor, up: int) -> torch.Tensor:
    """logits NHWC f32 [B, h, w, K] -> depth f32 [B, h up, w up] (no autograd)."""
    _need_cuda(logits, bins)
    logits, bins = logits.contiguous(), bins.contiguous()
    B, h, w, K = logits.shape
    if bins.numel() != K:
        raise DvtError(f"depth head: {bins.numel()} bins for {K} logits")
    out = torch.empty(B, h * up, w * up, device=logits.device, dtype=torch.float32)
    check(lib().dvt_depth_head_fwd(ptr(logits), B, h, w, K, int(up), ptr(bins), ptr(out), cur_stream()),
          "dvt_depth_head_fwd")
    return out


class _HeadDepth(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, bins, up):
        logits = logits.contiguous()
        ctx.save_for_backward(logits, bins)
        ctx.up = up
        return head_depth(logits, bins, up)

    @staticmethod
    def backward(ctx, g):
        logits, bins = ctx.saved_tensors
        g = g.contiguous()
        B, h, w, K = logits.shape
        dlogits = torch.empty_like(logits)
        check(lib().dvt_depth_head_bwd(ptr(logits), B, h, w, K, ctx.up, ptr(bins), ptr(g), ptr(dlogits), cur_stream()),
              "dvt_depth_head_bwd")
        return dlogits, None, None


def bin_expectation(logits: torch.Tensor, bins: torch.Tensor, up: int) -> torch.Tensor:
    """The head's depth at the upsampled grid, differentiable w.r.t. logits: the reference's
    einsum(normalise(relu(conv(resize(x, x up))) + 0.1), bins) with the conv taken at the feature grid."""
    return _HeadDepth.apply(logits, bins, int(up))


class _Resize(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, size):
        _need_cuda(x)
        x = x.contiguous()
        B, Hi, Wi = x.shape
        Ho, Wo = size
        ctx.shape = (B, Hi, Wi, Ho, Wo)
        out = torch.empty(B, Ho, Wo, device=x.device, dtype=torch.float32)
        check(lib().dvt_depth_resize_fwd(ptr(x), B, Hi, Wi, ptr(out), Ho, Wo, cur_stream()), "dvt_depth_resize_fwd")
        return out

    @staticmethod
    def backward(ctx, g):
        B, Hi, Wi, Ho, Wo = ctx.shape
        g = g.contiguous()
        din = torch.empty(B, Hi, Wi, device=g.device, dtype=torch.float32)
        check(lib().dvt_depth_resize_bwd(ptr(g), B, Hi, Wi, Ho, Wo, ptr(din), cur_stream()), "dvt_depth_resize_bwd")
        return din, None


def resize(x: torch.Tensor, size: Sequence[int]) -> torch.Tensor:
    """F.interpolate(x[:, None], size, bilinear, align_corners=False)[:, 0] for f32 [B, Hi, Wi], with a gather-form
    backward that torch.use_deterministic_algorithms accepts."""
    return _Resize.apply(x, (int(size[0]), int(size[1])))


# ---------------------------------------------------------------------------------------------------------------------
# losses on the [B, 1, H, W] prediction at the ground-truth size, as mask-multiplied ops (no boolean indexing, no host
# synchronisation)
# ---------------------------------------------------------------------------------------------------------------------
def sig_loss(pred: torch.Tensor, gt: torch.Tensor, warm_up: bool) -> torch.Tensor:
    """SigLoss(valid_mask=True): g = log(pred + eps) - log(gt + eps) over the pixels with gt > 0 of the whole batch;
    sqrt(var_unbiased(g) + 0.15 mean(g)^2), or sqrt(0.15 mean(g)^2) in warm-up."""
    m = (gt > 0).to(pred.dtype)
    n = m.sum()
    g = (torch.log(pred + LOSS_EPS) - torch.log(gt + LOSS_EPS)) * m
    mean = g.sum() / n
    if warm_up:
        return torch.sqrt(0.15 * mean * mean)
    var = (((g - mean) * m) ** 2).sum() / (n - 1)
    return torch.sqrt(var + 0.15 * mean * mean)


def gradient_loss(pred: torch.Tensor, gt: torch.Tensor) -> torch.Tensor:
    """GradientLoss(valid_mask=True) exactly as the reference writes it for 4-D [B, 1, H, W] tensors: the `[::2i, ::2i]`
    strides and the `[0:-2] - [2:]` differences act on the batch and channel dimensions, so the vertical term compares
    sample j with sample j + 2 and the horizontal one is empty.  It is 0 for a batch of 1 or 2 and NaN when a scale has
    no valid pixel."""
    total = pred.new_zeros(())
    for i in range(4):
        inp = pred if i == 0 else pred[::2 * i, ::2 * i]
        tgt = gt if i == 0 else gt[::2 * i, ::2 * i]
        mask = (tgt > 0).to(pred.dtype)
        n = mask.sum()
        ldd = (torch.log(inp + LOSS_EPS) - torch.log(tgt + LOSS_EPS)) * mask
        v = torch.abs(ldd[0:-2, :] - ldd[2:, :]) * (mask[0:-2, :] * mask[2:, :])
        h = torch.abs(ldd[:, 0:-2] - ldd[:, 2:]) * (mask[:, 0:-2] * mask[:, 2:])
        total = total + (h.sum() + v.sum()) / n
    return total


class SigLossState:
    """The reference SigLoss's warm-up: the first `warm_iter` calls in this process use the warm-up form.  The counter is
    module state that checkpoints do not hold, so a resumed run warms up again (a reference quirk kept on purpose)."""

    def __init__(self, warm_up: bool = True, warm_iter: int = 100):
        self.warm_up, self.warm_iter, self.counter = warm_up, warm_iter, 0

    def __call__(self, pred, gt):
        warm = self.warm_up and self.counter < self.warm_iter
        if warm:
            self.counter += 1
        return sig_loss(pred, gt, warm)


# ---------------------------------------------------------------------------------------------------------------------
# evaluation
# ---------------------------------------------------------------------------------------------------------------------
def eval_sums(maps: torch.Tensor, flips: Sequence[bool], gt: torch.Tensor, min_depth: float, max_depth: float,
              crop: Sequence[int], out: torch.Tensor, workspace: torch.Tensor) -> None:
    """maps f32 [n_aug, Hu, Wu] (one image), gt f32 [Ho, Wo], crop (y0, y1, x0, x1) -> out f64 [10] (see
    dvt_depth_eval_sums)."""
    _need_cuda(maps, gt)
    maps, gt = maps.contiguous(), gt.contiguous()
    n_aug, Hu, Wu = maps.shape
    if len(flips) != n_aug:
        raise DvtError(f"depth eval: {len(flips)} flip flags for {n_aug} maps")
    assert out.dtype == torch.float64 and out.numel() == 10 and workspace.dtype == torch.float64
    assert workspace.numel() >= EVAL_WORKSPACE and out.is_contiguous()
    mask = sum(1 << a for a, f in enumerate(flips) if f)
    y0, y1, x0, x1 = (int(v) for v in crop)
    check(lib().dvt_depth_eval_sums(ptr(maps), n_aug, mask, Hu, Wu, ptr(gt), gt.shape[0], gt.shape[1], float(min_depth),
                                    float(max_depth), y0, y1, x0, x1, ptr(workspace), ptr(out), cur_stream()),
          "dvt_depth_eval_sums")
