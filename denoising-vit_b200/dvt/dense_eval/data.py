"""Datasets and pipelines of the segmentation probe: mmseg 0.27's PascalVOCDataset / ADE20KDataset layouts and the train
and test pipelines of the linear configs, in numpy / PIL (and torch CPU resizes) inside DataLoader workers.

Restated from mmseg / mmcv, which cannot be installed beside this project, and so unpinned: mmcv decodes images with
OpenCV in BGR and resizes with cv2 (INTER_LINEAR, INTER_NEAREST for labels) and converts colour spaces with cv2.  Here
images are decoded by PIL in RGB (`to_rgb` is honoured by channel order), resized by torch's bilinear interpolation
with align_corners=False and no antialiasing (the sampling rule of cv2's INTER_LINEAR; cv2 rounds its fixed-point
weights differently) rounded back to uint8, labels by nearest-neighbour (floor(dst * in / out), as INTER_NEAREST), and
HSV is computed by the cv2 uint8 formulas restated in numpy.  Random draws follow mmseg's numpy.random call sequence,
from a RandomState per sample seeded by (seed, position in the sample stream), so a run does not depend on the number
of workers and a resumed run sees the samples the uninterrupted one would have seen."""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F
from PIL import Image

from .config import ConfigError

IGNORE = 255


# ---------------------------------------------------------------------------------------------------------------------
# geometry shared by the pipelines and slide inference
# ---------------------------------------------------------------------------------------------------------------------
def rescale_size(h: int, w: int, scale: Sequence[int]) -> Tuple[int, int]:
    """mmcv.imrescale with keep_ratio: the largest size that fits (long, short) edges `scale`, rounded half up."""
    long_edge, short_edge = max(scale), min(scale)
    f = min(long_edge / max(h, w), short_edge / min(h, w))
    return int(h * f + 0.5), int(w * f + 0.5)


def slide_windows(H: int, W: int, crop: Sequence[int], stride: Sequence[int]) -> List[Tuple[int, int, int, int]]:
    """mmseg EncoderDecoder.slide_inference window grid, in its order: (y1, y2, x1, x2) per window, rows outer."""
    h_crop, w_crop = crop
    h_stride, w_stride = stride
    h_grids = max(H - h_crop + h_stride - 1, 0) // h_stride + 1
    w_grids = max(W - w_crop + w_stride - 1, 0) // w_stride + 1
    out = []
    for hi in range(h_grids):
        for wi in range(w_grids):
            y1, x1 = hi * h_stride, wi * w_stride
            y2, x2 = min(y1 + h_crop, H), min(x1 + w_crop, W)
            out.append((max(y2 - h_crop, 0), y2, max(x2 - w_crop, 0), x2))
    return out


def resize_image(img: np.ndarray, size: Tuple[int, int]) -> np.ndarray:
    """uint8 HWC -> uint8 HWC of `size` (h, w): bilinear, align_corners=False, no antialiasing, rounded."""
    if img.shape[:2] == tuple(size):
        return img
    t = torch.from_numpy(np.ascontiguousarray(img)).permute(2, 0, 1)[None].float()
    t = F.interpolate(t, size=size, mode="bilinear", align_corners=False)
    return t[0].permute(1, 2, 0).round_().clamp_(0, 255).to(torch.uint8).numpy()


def resize_label(seg: np.ndarray, size: Tuple[int, int]) -> np.ndarray:
    if seg.shape[:2] == tuple(size):
        return seg
    t = torch.from_numpy(np.ascontiguousarray(seg))[None, None]
    return F.interpolate(t, size=size, mode="nearest")[0, 0].numpy()


def reduce_zero_label(seg: np.ndarray) -> np.ndarray:
    """ADE20K: class 0 ('other') becomes ignore, the others shift down by one."""
    seg = seg.copy()
    seg[seg == 0] = 255
    seg = seg - 1
    seg[seg == 254] = 255
    return seg


# ---------------------------------------------------------------------------------------------------------------------
# cv2's uint8 HSV conversion (H in [0, 180), S and V in [0, 255]) restated for RGB arrays
# ---------------------------------------------------------------------------------------------------------------------
def rgb2hsv(img: np.ndarray) -> np.ndarray:
    f = img.astype(np.float32)
    r, g, b = f[..., 0], f[..., 1], f[..., 2]
    v = f.max(-1)
    d = v - f.min(-1)
    safe = np.where(d > 0, d, 1.0)
    s = np.where(v > 0, d * 255.0 / np.where(v > 0, v, 1.0), 0.0)
    h = np.where(v == r, (g - b) * 60.0 / safe, np.where(v == g, 120.0 + (b - r) * 60.0 / safe,
                                                         240.0 + (r - g) * 60.0 / safe))
    h = np.where(d > 0, h, 0.0)
    h = np.where(h < 0, h + 360.0, h)
    out = np.stack([np.round(h / 2.0) % 180, np.round(s), v], -1)
    return out.astype(np.uint8)


def hsv2rgb(hsv: np.ndarray) -> np.ndarray:
    f = hsv.astype(np.float32)
    h, s, v = f[..., 0] * 2.0, f[..., 1] / 255.0, f[..., 2]
    c = v * s
    hp = h / 60.0
    x = c * (1.0 - np.abs(hp % 2.0 - 1.0))
    z = np.zeros_like(c)
    sector = np.floor(hp).astype(np.int64) % 6
    r = np.choose(sector, [c, x, z, z, x, c])
    g = np.choose(sector, [x, c, c, x, z, z])
    b = np.choose(sector, [z, z, x, c, c, x])
    m = v - c
    out = np.stack([r + m, g + m, b + m], -1)
    return np.clip(np.round(out), 0, 255).astype(np.uint8)


# ---------------------------------------------------------------------------------------------------------------------
# pipeline steps (mmseg/datasets/pipelines/transforms.py); each takes and returns a dict with `img` (HWC, RGB) and,
# in training, `seg` (HW uint8), and draws from `rng` in mmseg's order
# ---------------------------------------------------------------------------------------------------------------------
class Resize:
    def __init__(self, img_scale=None, ratio_range=None, keep_ratio=True, **kw):
        if not keep_ratio:
            raise ConfigError("Resize keep_ratio=False is not implemented")
        if kw.get("multiscale_mode", "range") != "range":
            raise ConfigError("Resize multiscale_mode is not implemented")
        self.img_scale = tuple(img_scale) if img_scale is not None else None
        self.ratio_range = tuple(ratio_range) if ratio_range is not None else None

    def __call__(self, r, rng):
        scale = r.get("scale", self.img_scale)     # `scale`: preset by a test-time augmentation, which draws nothing
        if "scale" not in r and self.ratio_range is not None:
            lo, hi = self.ratio_range
            ratio = rng.random_sample() * (hi - lo) + lo
            scale = int(self.img_scale[0] * ratio), int(self.img_scale[1] * ratio)
        size = rescale_size(r["img"].shape[0], r["img"].shape[1], scale)
        r["img"] = resize_image(r["img"], size)
        if "seg" in r:
            r["seg"] = resize_label(r["seg"], size)
        return r


class RandomCrop:
    def __init__(self, crop_size, cat_max_ratio=1.0, ignore_index=IGNORE):
        self.crop_size = tuple(crop_size)
        self.cat_max_ratio = cat_max_ratio
        self.ignore_index = ignore_index

    def bbox(self, img, rng):
        margin_h = max(img.shape[0] - self.crop_size[0], 0)
        margin_w = max(img.shape[1] - self.crop_size[1], 0)
        oh = rng.randint(0, margin_h + 1)
        ow = rng.randint(0, margin_w + 1)
        return oh, oh + self.crop_size[0], ow, ow + self.crop_size[1]

    def __call__(self, r, rng):
        box = self.bbox(r["img"], rng)
        if self.cat_max_ratio < 1.0:
            for _ in range(10):
                tmp = r["seg"][box[0]:box[1], box[2]:box[3]]
                labels, cnt = np.unique(tmp, return_counts=True)
                cnt = cnt[labels != self.ignore_index]
                if len(cnt) > 1 and np.max(cnt) / np.sum(cnt) < self.cat_max_ratio:
                    break
                box = self.bbox(r["img"], rng)
        r["img"] = r["img"][box[0]:box[1], box[2]:box[3]]
        for k in ("seg", "depth"):
            if k in r:
                r[k] = r[k][box[0]:box[1], box[2]:box[3]]
        return r


class RandomFlip:
    def __init__(self, prob=None, direction="horizontal"):
        if direction != "horizontal":
            raise ConfigError("RandomFlip: only horizontal flips are implemented")
        self.prob = prob

    def __call__(self, r, rng):
        if r["flip"] if "flip" in r else (self.prob is not None and rng.rand() < self.prob):
            r["img"] = r["img"][:, ::-1]
            for k in ("seg", "depth"):
                if k in r:
                    r[k] = r[k][:, ::-1]
        return r


class PhotoMetricDistortion:
    def __init__(self, brightness_delta=32, contrast_range=(0.5, 1.5), saturation_range=(0.5, 1.5), hue_delta=18):
        self.brightness_delta = brightness_delta
        self.contrast_lower, self.contrast_upper = contrast_range
        self.saturation_lower, self.saturation_upper = saturation_range
        self.hue_delta = hue_delta

    @staticmethod
    def convert(img, alpha=1.0, beta=0.0):
        return np.clip(img.astype(np.float32) * alpha + beta, 0, 255).astype(np.uint8)

    def __call__(self, r, rng):
        img = r["img"]
        if rng.randint(2):
            img = self.convert(img, beta=rng.uniform(-self.brightness_delta, self.brightness_delta))
        mode = rng.randint(2)
        if mode == 1 and rng.randint(2):
            img = self.convert(img, alpha=rng.uniform(self.contrast_lower, self.contrast_upper))
        if rng.randint(2):
            hsv = rgb2hsv(img)
            hsv[..., 1] = self.convert(hsv[..., 1], alpha=rng.uniform(self.saturation_lower, self.saturation_upper))
            img = hsv2rgb(hsv)
        if rng.randint(2):
            hsv = rgb2hsv(img)
            hsv[..., 0] = (hsv[..., 0].astype(int) + rng.randint(-self.hue_delta, self.hue_delta)) % 180
            img = hsv2rgb(hsv)
        if mode == 0 and rng.randint(2):
            img = self.convert(img, alpha=rng.uniform(self.contrast_lower, self.contrast_upper))
        r["img"] = img
        return r


class Normalize:
    def __init__(self, mean, std, to_rgb=True):
        self.mean = np.asarray(mean, np.float32)
        self.std = np.asarray(std, np.float32)
        self.to_rgb = to_rgb

    def __call__(self, r, rng):
        img = r["img"] if self.to_rgb else r["img"][..., ::-1]     # images are decoded as RGB
        r["img"] = (img.astype(np.float32) - self.mean) / self.std
        return r


class Pad:
    def __init__(self, size=None, pad_val=0, seg_pad_val=IGNORE, size_divisor=None):
        if size is None or size_divisor is not None:
            raise ConfigError("Pad: only a fixed `size` is implemented")
        self.size, self.pad_val, self.seg_pad_val = tuple(size), pad_val, seg_pad_val

    def __call__(self, r, rng):
        h, w = r["img"].shape[:2]
        H, W = max(h, self.size[0]), max(w, self.size[1])
        img = np.full((H, W) + r["img"].shape[2:], self.pad_val, dtype=r["img"].dtype)
        img[:h, :w] = r["img"]
        seg = np.full((H, W), self.seg_pad_val, dtype=np.uint8)
        seg[:h, :w] = r["seg"]
        r["img"], r["seg"] = img, seg
        return r


_STEPS = {"Resize": Resize, "RandomCrop": RandomCrop, "RandomFlip": RandomFlip,
          "PhotoMetricDistortion": PhotoMetricDistortion, "Normalize": Normalize, "Pad": Pad}
_NO_OP = ("LoadImageFromFile", "DefaultFormatBundle", "Collect", "ImageToTensor")


Aug = Tuple[Optional[Tuple[int, int]], bool]


def multiscale_flip_augs(kw: dict) -> List[Aug]:
    """mmseg MultiScaleFlipAug's augmentations, in its order (scale-major, then flip False, True): (scale (w, h), flip).
    With `img_ratios` the scales are (int(w * r), int(h * r)) of `img_scale` (w, h) for each ratio; without, `img_scale`
    itself.  One scale without flip (the linear configs) gives the single augmentation (img_scale, False)."""
    ratios, flip, scale = kw.get("img_ratios"), bool(kw.get("flip", False)), kw.get("img_scale")
    if not flip and (ratios is None or ratios in (1.0, [1.0], (1.0,))):
        return [(tuple(scale) if scale is not None else None, False)]
    if flip and kw.get("flip_direction", "horizontal") not in ("horizontal", ["horizontal"]):
        raise ConfigError(f"MultiScaleFlipAug flip_direction {kw.get('flip_direction')!r}: only horizontal flips are "
                          f"implemented")
    if ratios is not None:
        ratios = ratios if isinstance(ratios, list) else [ratios]
        if not all(isinstance(r, float) for r in ratios):
            raise ConfigError(f"MultiScaleFlipAug img_ratios {kw.get('img_ratios')!r}: a float or a list of floats")
        if scale is None:
            raise ConfigError("MultiScaleFlipAug img_ratios without img_scale (ratios of the image's own size) is not "
                              "implemented: give img_scale=(w, h)")
    if scale is None or len(scale) != 2 or not all(isinstance(v, (int, float)) for v in scale):
        raise ConfigError(f"MultiScaleFlipAug img_scale {scale!r}: only one (w, h) scale is implemented")
    scales = [(int(scale[0] * r), int(scale[1] * r)) for r in ratios] if ratios is not None else [tuple(scale)]
    return [(s, f) for s in scales for f in ((False, True) if flip else (False,))]


def build_pipeline(steps: List[dict], table: Optional[Dict[str, type]] = None) -> Tuple[list, bool, List[Aug]]:
    """(transforms, reduce_zero_label of LoadAnnotations, test-time augmentations).  MultiScaleFlipAug is flattened.
    With one augmentation its scale becomes the img_scale of an inner Resize without one.  With several, each
    augmentation runs the transforms with `scale` and `flip` preset; a pipeline without MultiScaleFlipAug has the single
    augmentation (None, False).  `table` maps step names to classes (default: the segmentation steps)."""
    table = _STEPS if table is None else table
    out, rzl, augs, outside = [], False, [(None, False)], 0
    for step in steps:
        kw = dict(step)
        t = kw.pop("type")
        if t in _NO_OP:
            continue
        if t == "LoadAnnotations":
            rzl = bool(kw.get("reduce_zero_label", False))
        elif t == "MultiScaleFlipAug":
            augs = multiscale_flip_augs(kw)
            inner, _, _ = build_pipeline(kw.get("transforms", []), table)
            if len(augs) == 1:
                for tr in inner:
                    if isinstance(tr, Resize) and tr.img_scale is None:
                        tr.img_scale = augs[0][0]
            out.extend(inner)
        elif t in table:
            out.append(table[t](**kw))
            outside += 1
        else:
            raise ConfigError(f"pipeline step {t!r} is not implemented")
    if len(augs) > 1 and outside:
        raise ConfigError("MultiScaleFlipAug with several augmentations: pipeline steps outside it are not implemented")
    return out, rzl, augs


# ---------------------------------------------------------------------------------------------------------------------
# datasets
# ---------------------------------------------------------------------------------------------------------------------
DATASET_DEFAULTS = {
    "PascalVOCDataset": dict(img_suffix=".jpg", seg_map_suffix=".png", reduce_zero_label=False),
    "ADE20KDataset": dict(img_suffix=".jpg", seg_map_suffix=".png", reduce_zero_label=True),
}


def _join(root, p):
    return p if (p is None or root is None or os.path.isabs(p)) else os.path.join(root, p)


def _load_image(path: str) -> np.ndarray:
    with Image.open(path) as im:
        return np.array(im.convert("RGB"))


def _load_label(path: str) -> np.ndarray:
    with Image.open(path) as im:       # palette PNGs give their indices, as mmcv's pillow backend
        return np.array(im, dtype=np.uint8)


class SegDataset(torch.utils.data.Dataset):
    """VOC layout (`split` file of names) or a sorted recursive listing of `img_dir` (ADE layout).

    Training (`train=True`): item t of the sample stream is image perm_e[t % n] of epoch e = t // n (a permutation drawn
    from `seed` + e), transformed with a RandomState seeded by (seed, t): returns (img f32 [3, H, W], seg u8 [H, W]).
    Evaluation: item i is image i after the test pipeline, with its ground truth at the original size (dataset-level
    reduce_zero_label applied): returns (img f32 [3, H, W], gt u8 [Ho, Wo]).  With several test-time augmentations
    (`augs`, mmseg's MultiScaleFlipAug order) it returns ([(img f32 [3, H_a, W_a], flip_a) per augmentation], gt)."""

    def __init__(self, ds_cfg: dict, num_classes: int, train: bool, seed: int = 0):
        d = dict(DATASET_DEFAULTS[ds_cfg["type"]])
        d.update({k: v for k, v in ds_cfg.items() if k in ("img_suffix", "seg_map_suffix", "reduce_zero_label")})
        root = ds_cfg.get("data_root")
        img_dir, ann_dir = _join(root, ds_cfg["img_dir"]), _join(root, ds_cfg.get("ann_dir"))
        split = _join(root, ds_cfg.get("split"))
        if split is not None:
            with open(split) as fh:
                names = [ln.strip() for ln in fh if ln.strip()]
            rel = [n + d["img_suffix"] for n in names]
        else:
            rel = sorted(os.path.relpath(os.path.join(dp, f), img_dir) for dp, _, fs in os.walk(img_dir, followlinks=True)
                         for f in fs if f.endswith(d["img_suffix"]))
        if not rel:
            raise FileNotFoundError(f"no images found under {img_dir}")
        self.images = [os.path.join(img_dir, r) for r in rel]
        self.labels = [os.path.join(ann_dir, r[:-len(d["img_suffix"])] + d["seg_map_suffix"]) for r in rel]
        self.transforms, self.pipeline_rzl, self.augs = build_pipeline(ds_cfg["pipeline"])
        self.reduce_zero_label = d["reduce_zero_label"]
        self.num_classes, self.train, self.seed = num_classes, train, seed
        self._perm = (None, None)

    def __len__(self):
        return len(self.images)

    def _check(self, seg, path):
        bad = (seg >= self.num_classes) & (seg != IGNORE)
        if bad.any():
            raise ValueError(f"{path}: label values {sorted(set(np.unique(seg[bad]).tolist()))} are neither < "
                             f"{self.num_classes} classes nor 255 (ignore)")

    def _index(self, t: int) -> int:
        n = len(self.images)
        epoch = t // n
        if self._perm[0] != epoch:
            self._perm = (epoch, np.random.RandomState((self.seed + epoch) % 2 ** 32).permutation(n))
        return int(self._perm[1][t % n])

    def __getitem__(self, t: int):
        i = self._index(t) if self.train else t
        img, seg = _load_image(self.images[i]), _load_label(self.labels[i])
        if self.train:
            if self.pipeline_rzl:
                seg = reduce_zero_label(seg)
            self._check(seg, self.labels[i])
            r = {"img": img, "seg": seg}
            rng = np.random.RandomState([self.seed % 2 ** 32, t])
            for tr in self.transforms:
                r = tr(r, rng)
            img_t = torch.from_numpy(np.ascontiguousarray(r["img"].transpose(2, 0, 1)))
            return img_t, torch.from_numpy(np.ascontiguousarray(r["seg"]))
        gt = reduce_zero_label(seg) if self.reduce_zero_label else seg
        self._check(gt, self.labels[i])
        gt = torch.from_numpy(np.ascontiguousarray(gt))
        if len(self.augs) > 1:
            return [(self._test_image(img, {"scale": scale, "flip": flip}), flip) for scale, flip in self.augs], gt
        return self._test_image(img, {}), gt

    def _test_image(self, img, preset):
        r = dict(preset, img=img)
        rng = np.random.RandomState(0)
        for tr in self.transforms:
            r = tr(r, rng)
        return torch.from_numpy(np.ascontiguousarray(r["img"].transpose(2, 0, 1)))


class StreamSampler(torch.utils.data.Sampler):
    """Positions in the training sample stream for iterations [start, stop) of one rank: iteration `it` of rank `r` takes
    positions (it * world + r) * batch + j, j < batch."""

    def __init__(self, start: int, stop: int, batch: int, rank: int = 0, world: int = 1):
        self.start, self.stop, self.batch, self.rank, self.world = start, stop, batch, rank, world

    def __iter__(self):
        for it in range(self.start, self.stop):
            base = (it * self.world + self.rank) * self.batch
            yield from range(base, base + self.batch)

    def __len__(self):
        return (self.stop - self.start) * self.batch


def worker_init_fn(worker_id: int, num_workers: int, rank: int, seed: int):
    """mmseg's per-worker seeding (num_workers * rank + worker_id + seed) for any draw outside the per-sample RNG."""
    s = (num_workers * rank + worker_id + seed) % 2 ** 32
    np.random.seed(s)
    torch.manual_seed(s)
    torch.set_num_threads(1)
