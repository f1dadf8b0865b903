"""torch bindings of the segmentation-probe kernels (include/dvt_b200.h, `dvt_seg_*`)."""
from __future__ import annotations

from typing import Sequence, Tuple

import torch

from .._lib import DvtError, check, cur_stream, lib, ptr


def _need_cuda(*ts):
    for t in ts:
        if not t.is_cuda:
            raise DvtError("dvt_b200 segmentation kernels need CUDA tensors (no CPU fallback)")


def upsample_ce_sum(logits: torch.Tensor, labels: torch.Tensor, grad_scale: float) -> Tuple[torch.Tensor, torch.Tensor]:
    """logits f32 [B, h, w, K] (NHWC), labels u8 [B, H, W] -> (sum of the per-pixel cross-entropy of the bilinearly
    upsampled logits, f32 [1]; grad_scale * its gradient w.r.t. logits, f32 [B, h, w, K])."""
    _need_cuda(logits, labels)
    if logits.dtype != torch.float32 or labels.dtype != torch.uint8:
        raise DvtError("upsample_ce: logits must be float32 and labels uint8")
    logits, labels = logits.contiguous(), labels.contiguous()
    B, h, w, K = logits.shape
    H, W = labels.shape[1:]
    if labels.shape[0] != B:
        raise DvtError(f"upsample_ce: {B} logit maps but {labels.shape[0]} label maps")
    loss = torch.empty(1, device=logits.device, dtype=torch.float32)
    dlogits = torch.empty_like(logits)
    ws = torch.empty(B * ((h + 1) // 2) * ((w + 1) // 2), device=logits.device, dtype=torch.float64)
    check(lib().dvt_seg_upsample_ce(ptr(logits), B, h, w, K, ptr(labels), H, W, float(grad_scale), ptr(loss), ptr(dlogits),
                                    ptr(ws), cur_stream()), "dvt_seg_upsample_ce")
    return loss, dlogits


class _UpsampleCE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, labels):
        n = labels.numel()
        loss, dlogits = upsample_ce_sum(logits, labels, 1.0 / n)
        ctx.save_for_backward(dlogits)
        return loss[0] / n

    @staticmethod
    def backward(ctx, g):
        (dlogits,) = ctx.saved_tensors
        return dlogits * g, None


def upsample_cross_entropy(logits: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
    """mmseg's decode-head loss: resize(logits, label size, bilinear, align_corners=False) then CrossEntropyLoss with
    ignore_index 255 and the mean over ALL pixels (mmseg 0.27's avg_non_ignore=False).  logits NHWC [B, h, w, K].  The
    forward computes the low-resolution gradient too (one kernel); the backward only scales it."""
    return _UpsampleCE.apply(logits, labels)


def slide_accumulate(logits_hwk: torch.Tensor, y1: int, x1: int, wh: int, ww: int, acc: torch.Tensor,
                     count: torch.Tensor) -> None:
    """acc [K, Hc, Wc] += resize(logits [h, w, K] -> wh x ww) at (y1, x1); count [Hc, Wc] += 1 there."""
    _need_cuda(logits_hwk, acc, count)
    h, w, K = logits_hwk.shape
    assert logits_hwk.is_contiguous() and acc.is_contiguous() and count.is_contiguous() and acc.shape[0] == K
    check(lib().dvt_seg_slide_accumulate(ptr(logits_hwk), h, w, K, y1, x1, wh, ww, ptr(acc), ptr(count), acc.shape[1],
                                         acc.shape[2], cur_stream()), "dvt_seg_slide_accumulate")


def predict_hist(acc: torch.Tensor, count: torch.Tensor, labels: torch.Tensor, hist: torch.Tensor) -> None:
    """acc /= count (in place), resize to the label size, argmax, hist int64 [4, K] += (intersect, union, pred, label)."""
    _need_cuda(acc, count, labels, hist)
    K, Hc, Wc = acc.shape
    assert labels.dtype == torch.uint8 and labels.is_contiguous() and hist.dtype == torch.int64 and hist.shape == (4, K)
    check(lib().dvt_seg_predict_hist(ptr(acc), ptr(count), K, Hc, Wc, ptr(labels), labels.shape[0], labels.shape[1],
                                     ptr(hist), cur_stream()), "dvt_seg_predict_hist")


def slide_inference_hist(logits_fn, img: torch.Tensor, gt: torch.Tensor, num_classes: int, crop: Sequence[int],
                         stride: Sequence[int], hist: torch.Tensor, max_batch: int = 8) -> None:
    """mmseg slide inference of one normalised image img [3, H, W] followed by the histograms of its prediction against
    gt u8 [Ho, Wo] (the original size).  `logits_fn(crops [n, 3, wh, ww]) -> [n, h, w, K]` NHWC logits; windows go
    through it in batches of `max_batch` and are accumulated in mmseg's order."""
    from .data import slide_windows
    H, W = img.shape[1:]
    wins = slide_windows(H, W, crop, stride)
    acc = torch.zeros(num_classes, H, W, device=img.device, dtype=torch.float32)
    count = torch.zeros(H, W, device=img.device, dtype=torch.float32)
    for s in range(0, len(wins), max_batch):
        chunk = wins[s:s + max_batch]
        crops = torch.stack([img[:, y1:y2, x1:x2] for (y1, y2, x1, x2) in chunk])
        logits = logits_fn(crops).contiguous()
        for j, (y1, y2, x1, x2) in enumerate(chunk):
            slide_accumulate(logits[j], y1, x1, y2 - y1, x2 - x1, acc, count)
    predict_hist(acc, count, gt, hist)
