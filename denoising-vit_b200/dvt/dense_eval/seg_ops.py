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


def aug_accumulate(acc: torch.Tensor, count: torch.Tensor, flip: bool, prob: torch.Tensor) -> None:
    """prob [K, Ho, Wo] += un-flip(softmax over K of resize(acc [K, Hc, Wc] / count [Hc, Wc] -> Ho x Wo)); the un-flip is
    horizontal and applies when `flip` is set.  acc and count are not written."""
    _need_cuda(acc, count, prob)
    K, Hc, Wc = acc.shape
    assert acc.is_contiguous() and count.is_contiguous() and prob.is_contiguous() and prob.shape[0] == K
    assert acc.dtype == count.dtype == prob.dtype == torch.float32 and count.shape == (Hc, Wc)
    check(lib().dvt_seg_aug_accumulate(ptr(acc), ptr(count), K, Hc, Wc, int(bool(flip)), ptr(prob), prob.shape[1],
                                       prob.shape[2], cur_stream()), "dvt_seg_aug_accumulate")


def aug_argmax_hist(prob: torch.Tensor, n_aug: int, labels: torch.Tensor, hist: torch.Tensor) -> None:
    """argmax over K of prob [K, Ho, Wo] / n_aug, hist int64 [4, K] += (intersect, union, pred, label)."""
    _need_cuda(prob, labels, hist)
    K = prob.shape[0]
    assert prob.dtype == torch.float32 and prob.is_contiguous() and prob.shape[1:] == labels.shape
    assert labels.dtype == torch.uint8 and labels.is_contiguous() and hist.dtype == torch.int64 and hist.shape == (4, K)
    check(lib().dvt_seg_aug_argmax_hist(ptr(prob), int(n_aug), K, ptr(labels), labels.shape[0], labels.shape[1], ptr(hist),
                                        cur_stream()), "dvt_seg_aug_argmax_hist")


def aug_slide_inference_hist(logits_fn, augs: Sequence[Tuple[torch.Tensor, bool]], gt: torch.Tensor, num_classes: int,
                             crop: Sequence[int], stride: Sequence[int], hist: torch.Tensor, max_batch: int = 8) -> None:
    """mmseg aug_test of one image followed by the histograms of its prediction against gt u8 [Ho, Wo] (the original
    size).  `augs` lists (normalised image [3, H, W], flip) per augmentation, in mmseg's order.  Each augmentation is slide
    inference at its own size, then the resize of preds / count to Ho x Wo, softmax and un-flip, summed in augmentation
    order; the sum / len(augs) gives the argmax.  Windows go through `logits_fn` (as in `slide_inference_hist`) in
    batches of up to `max_batch` consecutive windows of one shape, across augmentations; an augmentation's
    accumulators are released once its last window is added."""
    from .data import slide_windows
    K = num_classes
    prob = torch.zeros(K, *gt.shape, device=gt.device, dtype=torch.float32)
    jobs = [(a, win) for a, (img, _) in enumerate(augs) for win in slide_windows(img.shape[1], img.shape[2], crop, stride)]
    last = {a: j for j, (a, _) in enumerate(jobs)}
    bufs = {}
    s = 0
    while s < len(jobs):
        shape = _win_shape(jobs[s][1])
        e = s + 1
        while e < len(jobs) and e - s < max_batch and _win_shape(jobs[e][1]) == shape:
            e += 1
        crops = torch.stack([augs[a][0][:, y1:y2, x1:x2] for a, (y1, y2, x1, x2) in jobs[s:e]])
        logits = logits_fn(crops).contiguous()
        for j in range(s, e):
            a, (y1, y2, x1, x2) = jobs[j]
            img, flip = augs[a]
            if a not in bufs:
                bufs[a] = (torch.zeros(K, img.shape[1], img.shape[2], device=img.device, dtype=torch.float32),
                           torch.zeros(img.shape[1], img.shape[2], device=img.device, dtype=torch.float32))
            acc, count = bufs[a]
            slide_accumulate(logits[j - s], y1, x1, y2 - y1, x2 - x1, acc, count)
            if j == last[a]:
                aug_accumulate(acc, count, flip, prob)
                del bufs[a]
        s = e
    aug_argmax_hist(prob, len(augs), gt, hist)


def _win_shape(win):
    y1, y2, x1, x2 = win
    return y2 - y1, x2 - x1


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
