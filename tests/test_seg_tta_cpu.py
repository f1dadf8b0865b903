"""Segmentation probe, test-time augmentation without a GPU: MultiScaleFlipAug's augmentation list (scales, order, flip
flags) and the image sizes it gives, against hand-computed int(w * r) / keep-ratio sizes; the refusals; the evaluation
dataset's augmented images; and the reference configs still giving one augmentation and today's tensors."""
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

from dvt.dense_eval import config as C  # noqa: E402
from dvt.dense_eval import data as D  # noqa: E402

RATIOS = [0.5, 0.75, 1.0, 1.25, 1.5, 1.75]
MS_FLIP = {"data.val.pipeline.1.img_ratios": RATIOS, "data.val.pipeline.1.flip": True}
MEAN, STD = [123.675, 116.28, 103.53], [58.395, 57.12, 57.375]


def _gold(name):
    with open(os.path.join(GOLDEN, "dense_eval_configs.json")) as fh:
        return json.load(fh)[name]


def _msfa(**kw):
    step = {"type": "MultiScaleFlipAug", "img_scale": (2048, 512),
            "transforms": [{"type": "Resize", "keep_ratio": True}, {"type": "RandomFlip"},
                           {"type": "Normalize", "mean": MEAN, "std": STD, "to_rgb": True},
                           {"type": "ImageToTensor", "keys": ["img"]}, {"type": "Collect", "keys": ["img"]}]}
    step.update(kw)
    return [{"type": "LoadImageFromFile"}, step]


def test_six_ratios_with_flip_in_mmseg_order():
    _, _, augs = D.build_pipeline(_msfa(img_ratios=RATIOS, flip=True))
    # (int(2048 r), int(512 r)) per ratio, scale-major, then flip False, True
    scales = [(1024, 256), (1536, 384), (2048, 512), (2560, 640), (3072, 768), (3584, 896)]
    assert augs == [(s, f) for s in scales for f in (False, True)]
    _, _, augs = D.build_pipeline(_msfa(img_ratios=[0.5, 1.0]))
    assert augs == [((1024, 256), False), ((2048, 512), False)]
    _, _, augs = D.build_pipeline(_msfa(flip=True))
    assert augs == [((2048, 512), False), ((2048, 512), True)]
    _, _, augs = D.build_pipeline(_msfa(img_ratios=0.75, flip=True, img_scale=[1001, 333]))
    assert augs == [((750, 249), False), ((750, 249), True)]


@pytest.mark.parametrize("h, w, sizes", [
    # keep-ratio fit of (h, w) into each scale's (long, short) edges, rounded half up
    (375, 500, [(256, 341), (384, 512), (512, 683), (640, 853), (768, 1024), (896, 1195)]),
    (512, 2048, [(256, 1024), (384, 1536), (512, 2048), (640, 2560), (768, 3072), (896, 3584)]),
    (333, 500, [(256, 384), (384, 577), (512, 769), (640, 961), (768, 1153), (896, 1345)]),
    (101, 1000, [(103, 1024), (155, 1536), (207, 2048), (259, 2560), (310, 3072), (362, 3584)]),
])
def test_augmented_image_sizes_and_flips(tmp_path, h, w, sizes):
    root = _voc(tmp_path, [(h, w)])
    cfg = _voc_cfg(root, MS_FLIP)
    ds = D.SegDataset(cfg["data"]["val"], 21, train=False)
    views, gt = ds[0]
    assert gt.shape == (h, w) and gt.dtype == torch.uint8
    assert [tuple(v.shape[1:]) for v, _ in views] == [s for s in sizes for _ in (0, 1)]
    assert [f for _, f in views] == [False, True] * 6
    for (a, _), (b, _) in zip(views[0::2], views[1::2]):
        assert a.dtype == torch.float32 and torch.equal(a.flip(2), b)
    # the unflipped ratio-1.0 view is the single-scale image
    single, gt1 = D.SegDataset(_voc_cfg(root, {})["data"]["val"], 21, train=False)[0]
    assert torch.equal(views[4][0], single) and torch.equal(gt, gt1)


@pytest.mark.parametrize("kw, msg", [
    (dict(img_ratios=RATIOS, img_scale=None), "img_scale"),
    (dict(img_ratios=0.5, flip=True, img_scale=None), "img_scale"),
    (dict(flip=True, flip_direction="vertical"), "flip_direction"),
    (dict(flip=True, flip_direction=["horizontal", "vertical"]), "flip_direction"),
    (dict(img_ratios=[1, 2]), "img_ratios"),
    (dict(img_ratios=[0.5, 1]), "img_ratios"),
    (dict(img_ratios=(0.5, 1.0)), "img_ratios"),
    (dict(img_ratios=2, flip=True), "img_ratios"),
    (dict(flip=True, img_scale=[(2048, 512), (1024, 256)]), "img_scale"),
])
def test_refusals(kw, msg):
    with pytest.raises(C.ConfigError, match=msg):
        D.build_pipeline(_msfa(**kw))


def test_steps_outside_a_multi_augmentation_are_refused():
    steps = _msfa(img_ratios=RATIOS) + [{"type": "Normalize", "mean": MEAN, "std": STD}]
    with pytest.raises(C.ConfigError, match="outside"):
        D.build_pipeline(steps)


@pytest.mark.parametrize("name", ["vitb_voc2012_linear_config.py", "vitb_ade20k_linear_config.py"])
def test_reference_configs_keep_one_augmentation_and_their_tensors(tmp_path, name):
    gold = _gold(name)
    steps = gold["data"]["val"]["pipeline"]
    transforms, rzl, augs = D.build_pipeline(steps)
    assert augs == [((2048, 512), False)] and rzl is False
    assert [type(t).__name__ for t in transforms] == ["Resize", "RandomFlip", "Normalize"]
    assert transforms[0].img_scale == (2048, 512) and transforms[1].prob is None
    _, _, train_augs = D.build_pipeline(gold["data"]["train"]["pipeline"])
    assert train_augs == [(None, False)]
    root = _voc(tmp_path, [(375, 500), (90, 130)])
    cfg = _voc_cfg(root, {"data.val.pipeline": steps})
    ds = D.SegDataset(cfg["data"]["val"], 21, train=False)
    assert ds.augs == [((2048, 512), False)]
    for i, (h, w) in enumerate([(375, 500), (90, 130)]):
        img, gt = ds[i]
        # the single-scale test pipeline: keep-ratio resize into (2048, 512), no flip, normalise
        raw = D._load_image(ds.images[i])
        ref = (D.resize_image(raw, D.rescale_size(h, w, (2048, 512))).astype(np.float32) - np.float32(MEAN)) / np.float32(STD)
        assert isinstance(img, torch.Tensor) and torch.equal(img, torch.from_numpy(np.ascontiguousarray(ref.transpose(2, 0, 1))))
        assert torch.equal(gt, torch.from_numpy(D._load_label(ds.labels[i])))


def test_cfg_options_enable_ms_flip():
    sys.path.insert(0, ROOT)
    import evaluate_dense_tasks as E
    a = E.parse_args(["cfg.py", "--cfg-options", "data.val.pipeline.1.img_ratios=[0.5,0.75,1.0,1.25,1.5,1.75]",
                      "data.val.pipeline.1.flip=True"])
    assert a.cfg_options == MS_FLIP
    cfg = C.merge_options(_gold("vitb_ade20k_linear_config.py"), a.cfg_options)
    C.check_supported(cfg)
    _, _, augs = D.build_pipeline(cfg["data"]["val"]["pipeline"])
    assert len(augs) == 12 and augs[5] == ((2048, 512), True)


def test_preset_flip_and_scale_draw_nothing():
    img = np.arange(4 * 6 * 3, dtype=np.uint8).reshape(4, 6, 3)
    rng = np.random.RandomState(0)
    r = D.RandomFlip(prob=0.5)({"img": img, "flip": True}, rng)
    r = D.Resize(img_scale=(2048, 512), ratio_range=(0.5, 2.0))(dict(r, scale=(12, 8)), rng)
    assert r["img"].shape == (8, 12, 3)
    assert rng.rand() == np.random.RandomState(0).rand()
    r = D.RandomFlip()({"img": img, "flip": False}, rng)
    assert np.array_equal(r["img"], img)


def test_tta_ops_refuse_cpu_tensors():
    from dvt._lib import DvtError
    from dvt.dense_eval import seg_ops
    acc, count, prob = torch.zeros(3, 4, 5), torch.ones(4, 5), torch.zeros(3, 6, 7)
    with pytest.raises(DvtError):
        seg_ops.aug_accumulate(acc, count, True, prob)
    with pytest.raises(DvtError):
        seg_ops.aug_argmax_hist(prob, 2, torch.zeros(6, 7, dtype=torch.uint8), torch.zeros(4, 3, dtype=torch.int64))


# ---------------------------------------------------------------------------------------------------------------------
def _voc(root, shapes):
    """VOC layout with one random image (and label map) per (h, w)."""
    from PIL import Image
    for d in ("JPEGImages", "SegmentationClass", "ImageSets/Segmentation"):
        (root / d).mkdir(parents=True, exist_ok=True)
    rs = np.random.RandomState(0)
    names = []
    for i, (h, w) in enumerate(shapes):
        name = f"img{i:03d}"
        Image.fromarray(rs.randint(0, 256, (h, w, 3)).astype(np.uint8)).save(root / "JPEGImages" / f"{name}.jpg")
        Image.fromarray(rs.randint(0, 21, (h, w)).astype(np.uint8)).save(root / "SegmentationClass" / f"{name}.png")
        names.append(name)
    (root / "ImageSets/Segmentation/val.txt").write_text("\n".join(names) + "\n")
    return root


def _voc_cfg(root, options):
    cfg = _gold("vitb_voc2012_linear_config.py")
    return C.merge_options(cfg, dict({"data.val.data_root": str(root)}, **options))
