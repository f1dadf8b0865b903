"""mmseg 0.27 `total_area_to_metrics` for mIoU: dataset-wide histograms -> aAcc, mIoU, mAcc and per-class IoU / Acc.

The histograms are the int64 [4, K] rows (intersect, union, pred, label) that `dvt_seg_predict_hist` accumulates.  Values
are fractions in [0, 1] (mmseg logs them as rounded percentages); a class absent from both prediction and ground truth
has IoU NaN and a class absent from the ground truth has Acc NaN, and the means skip NaNs (np.nanmean)."""
from __future__ import annotations

import warnings
from typing import Dict

import numpy as np


def metrics_from_hist(hist) -> Dict[str, object]:
    h = np.asarray(hist, dtype=np.float64)
    inter, union, label = h[0], h[1], h[3]
    with np.errstate(divide="ignore", invalid="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)
        iou = inter / union
        acc = inter / label
        return {"aAcc": float(inter.sum() / label.sum()), "mIoU": float(np.nanmean(iou)), "mAcc": float(np.nanmean(acc)),
                "IoU": [None if np.isnan(v) else float(v) for v in iou],
                "Acc": [None if np.isnan(v) else float(v) for v in acc]}
