"""NYU-Depth dataset and the pipeline steps of the depth probe (reference evaluation/depth/datasets/nyu.py and
pipelines/transforms.py), in numpy / PIL inside DataLoader workers.

Restated from mmcv / mmseg-based code that cannot be installed beside this project, and so unpinned, like the
segmentation pipelines (data.py).  The reference decodes BGR with cv2; here PIL decodes RGB, so ColorAug's per-channel
factor colors[i] (drawn for BGR channel i) multiplies RGB channel 2 - i.  RandomRotate restates cv2.warpAffine with the
matrix of mmcv.imrotate (cv2.getRotationMatrix2D(center, -angle, 1), centre ((w - 1) / 2, (h - 1) / 2), constant border
0): bilinear for the image with float weights (cv2 quantises them to 1/32) rounded back to uint8, nearest
(floor(src + 0.5)) for the depth.  `Normalize`, `RandomFlip`, `RandomCrop`, the sample stream and the worker seeding are
the segmentation probe's; random draws follow the reference's numpy.random call sequence from a RandomState per sample
seeded by (seed, position in the sample stream)."""
from __future__ import annotations

import math
import os
from typing import List, Tuple

import numpy as np
import torch
from PIL import Image

from .config import ConfigError
from .data import Normalize, RandomCrop, RandomFlip, SegDataset, build_pipeline


class NYUCrop:
    """Image and depth rows 45:472, columns 43:608 (the NYU border without depth)."""

    def __init__(self, depth=False):
        self.depth = depth

    def __call__(self, r, rng):
        r["img"] = r["img"][45:472, 43:608]
        if self.depth and "depth" in r:
            r["depth"] = r["depth"][45:472, 43:608]
        return r


def rotation_source(h: int, w: int, degree: float) -> Tuple[np.ndarray, np.ndarray]:
    """Source coordinates (sx, sy) [h, w] of every destination pixel of mmcv.imrotate(angle=degree) (no auto_bound)."""
    cx, cy = (w - 1) * 0.5, (h - 1) * 0.5
    t = math.radians(-degree)
    a, b = math.cos(t), math.sin(t)
    t0, t1 = (1 - a) * cx - b * cy, b * cx + (1 - a) * cy     # cv2.getRotationMatrix2D(center, -degree, 1)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    return a * (x - t0) - b * (y - t1), b * (x - t0) + a * (y - t1)  # the inverse of [[a, b], [-b, a]]


def rotate_bilinear(img: np.ndarray, degree: float, border=0) -> np.ndarray:
    h, w = img.shape[:2]
    sx, sy = rotation_source(h, w, degree)
    x0, y0 = np.floor(sx).astype(np.int64), np.floor(sy).astype(np.int64)
    fx, fy = (sx - x0)[..., None], (sy - y0)[..., None]
    f = img.reshape(h, w, -1).astype(np.float64)

    def tap(yy, xx):
        ok = (yy >= 0) & (yy < h) & (xx >= 0) & (xx < w)
        v = f[np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)]
        return np.where(ok[..., None], v, float(border))

    out = ((1 - fy) * ((1 - fx) * tap(y0, x0) + fx * tap(y0, x0 + 1)) +
           fy * ((1 - fx) * tap(y0 + 1, x0) + fx * tap(y0 + 1, x0 + 1)))
    if img.dtype == np.uint8:
        out = np.clip(np.floor(out + 0.5), 0, 255)
    return out.astype(img.dtype).reshape(img.shape)


def rotate_nearest(img: np.ndarray, degree: float, border=0) -> np.ndarray:
    h, w = img.shape[:2]
    sx, sy = rotation_source(h, w, degree)
    xi, yi = np.floor(sx + 0.5).astype(np.int64), np.floor(sy + 0.5).astype(np.int64)
    ok = (yi >= 0) & (yi < h) & (xi >= 0) & (xi < w)
    return np.where(ok, img[np.clip(yi, 0, h - 1), np.clip(xi, 0, w - 1)], border).astype(img.dtype)


class RandomRotate:
    """Draws rand() and then uniform(-degree, degree) on every call (the reference draws the angle even when it does not
    rotate); rotates with probability `prob`."""

    def __init__(self, prob, degree, pad_val=0, depth_pad_val=0, center=None, auto_bound=False):
        if center is not None or auto_bound:
            raise ConfigError("RandomRotate: only the default centre without auto_bound is implemented")
        self.prob = prob
        self.degree = (-degree, degree) if isinstance(degree, (int, float)) else tuple(degree)
        self.pad_val, self.depth_pad_val = pad_val, depth_pad_val

    def __call__(self, r, rng):
        rotate = rng.rand() < self.prob
        degree = rng.uniform(min(*self.degree), max(*self.degree))
        if rotate:
            r["img"] = rotate_bilinear(r["img"], degree, self.pad_val)
            if "depth" in r:
                r["depth"] = rotate_nearest(r["depth"], degree, self.depth_pad_val)
        return r


class ColorAug:
    """With probability `prob`: img ** gamma * brightness * colors (per channel), clipped to [0, 255], in float64."""

    def __init__(self, prob=None, gamma_range=(0.9, 1.1), brightness_range=(0.9, 1.1), color_range=(0.9, 1.1)):
        self.prob = prob
        self.gamma_range, self.brightness_range, self.color_range = gamma_range, brightness_range, color_range

    def __call__(self, r, rng):
        if rng.rand() < self.prob:
            img = r["img"]
            gamma = rng.uniform(min(*self.gamma_range), max(*self.gamma_range))
            aug = img ** gamma
            aug = aug * rng.uniform(min(*self.brightness_range), max(*self.brightness_range))
            colors = rng.uniform(min(*self.color_range), max(*self.color_range), size=3)
            aug = aug * colors[::-1][None, None, :]    # BGR draw order, RGB image
            r["img"] = np.clip(aug, 0, 255)
        return r


class _NoOp:
    def __init__(self, **kw):
        pass

    def __call__(self, r, rng):
        return r


DEPTH_STEPS = {"NYUCrop": NYUCrop, "RandomRotate": RandomRotate, "RandomFlip": RandomFlip, "RandomCrop": RandomCrop,
               "ColorAug": ColorAug, "Normalize": Normalize, "DepthLoadAnnotations": _NoOp}


def _strip(s: str) -> str:
    return s[1:] if s[:1] in ("/", "\\") else s


def parse_split(path: str, data_root: str) -> List[Tuple[str, str]]:
    """(image, depth) paths of a `rgb depth focal` split file: lines whose depth is `None` are skipped, the leading
    slash is stripped and the path joined to data_root; sorted by image path."""
    out = []
    with open(path) as fh:
        for line in fh:
            if not line.strip():
                continue
            parts = line.strip().split(" ")
            if parts[1] == "None":
                continue
            out.append((os.path.join(data_root, _strip(parts[0])), os.path.join(data_root, _strip(parts[1]))))
    return sorted(out, key=lambda p: p[0])


def load_depth(path: str, depth_scale: float) -> np.ndarray:
    with Image.open(path) as im:
        return np.asarray(im, dtype=np.float32) / depth_scale


class NYUDataset(torch.utils.data.Dataset):
    """Training (`train=True`): item t of the sample stream is image perm_e[t % n] of epoch e = t // n, transformed with
    a RandomState seeded by (seed, t): (img f32 [3, H, W], depth f32 [H, W]).  Evaluation: item i is image i under each
    test-time augmentation: ([(img f32 [3, H, W], flip)], depth f32 [Ho, Wo] at the original size)."""

    _index = SegDataset._index

    def __init__(self, ds_cfg: dict, train: bool, seed: int = 0):
        root = ds_cfg.get("data_root") or ""
        split = ds_cfg["split"]
        split = split if os.path.isabs(split) else os.path.join(root, split)
        pairs = parse_split(split, root)
        if not pairs:
            raise FileNotFoundError(f"no images listed in {split}")
        self.images, self.depths = [p[0] for p in pairs], [p[1] for p in pairs]
        self.depth_scale = float(ds_cfg.get("depth_scale", 1000))
        self.min_depth, self.max_depth = float(ds_cfg.get("min_depth", 1e-3)), float(ds_cfg.get("max_depth", 10))
        self.garg_crop, self.eigen_crop = bool(ds_cfg.get("garg_crop", False)), bool(ds_cfg.get("eigen_crop", True))
        self.transforms, _, self.augs = build_pipeline(ds_cfg["pipeline"], DEPTH_STEPS)
        self.train, self.seed = train, seed
        self._perm = (None, None)

    def __len__(self):
        return len(self.images)

    def eval_crop(self, h: int, w: int) -> Tuple[int, int, int, int]:
        """(y0, y1, x0, x1) of NYUDataset.eval_mask: the garg crop, else the eigen crop [45:471, 41:601], else all."""
        if self.garg_crop:
            return int(0.40810811 * h), int(0.99189189 * h), int(0.03594771 * w), int(0.96405229 * w)
        if self.eigen_crop:
            return 45, 471, 41, 601
        return 0, h, 0, w

    def __getitem__(self, t: int):
        i = self._index(t) if self.train else t
        with Image.open(self.images[i]) as im:
            img = np.array(im.convert("RGB"))
        depth = load_depth(self.depths[i], self.depth_scale)
        if self.train:
            r = {"img": img, "depth": depth}
            rng = np.random.RandomState([self.seed % 2 ** 32, t])
            for tr in self.transforms:
                r = tr(r, rng)
            return (torch.from_numpy(np.ascontiguousarray(r["img"].transpose(2, 0, 1))),
                    torch.from_numpy(np.ascontiguousarray(r["depth"])))
        augs = []
        for _, flip in self.augs:
            r = {"img": img, "flip": flip}
            rng = np.random.RandomState(0)
            for tr in self.transforms:
                r = tr(r, rng)
            augs.append((torch.from_numpy(np.ascontiguousarray(r["img"].transpose(2, 0, 1))), flip))
        return augs, torch.from_numpy(np.ascontiguousarray(depth))
