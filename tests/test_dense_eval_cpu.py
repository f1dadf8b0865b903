"""Segmentation probe without a GPU: the CLI's flags against the reference parser (golden read with ast), the config
loader against the executed reference configs (golden JSON), and the host-side pieces -- keep-ratio resize, slide-window
grid, pipeline steps, LR schedule, metrics -- against hand-computed values."""
import json
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")

from dvt.dense_eval import config as C  # noqa: E402
from dvt.dense_eval import data as D  # noqa: E402
from dvt.dense_eval.metrics import metrics_from_hist  # noqa: E402
from dvt.dense_eval.trainer import poly_lr  # noqa: E402


def _jsonable(v):
    if isinstance(v, dict):
        return {k: _jsonable(x) for k, x in v.items()}
    if isinstance(v, (list, tuple, range)):
        return [_jsonable(x) for x in v]
    return v


def test_cli_flags_match_the_reference():
    sys.path.insert(0, GOLDEN)
    try:
        from make_cli_golden import flags
    finally:
        sys.path.pop(0)
    with open(os.path.join(GOLDEN, "cli_flags_dense_eval.json")) as fh:
        ref = json.load(fh)["evaluate_dense_tasks.py"]
    ours = flags(os.path.join(ROOT, "evaluate_dense_tasks.py"))
    assert len(ref) == 17 and "--load-denoiser-from" in ref and "--cfg-options" in ref
    for name, spec in ref.items():
        assert ours.get(name) == spec, f"{name}: {ours.get(name)} != reference {spec}"


def test_cli_parses_and_refuses_depth(tmp_path):
    sys.path.insert(0, ROOT)
    import evaluate_dense_tasks as E
    a = E.parse_args(["cfg.py", "--cfg-options", "runner.max_iters=10", "model.decode_head.in_index=[3]",
                      "data.samples_per_gpu=4"])
    assert a.launcher == "pytorch" and a.seed is None and a.num_blocks == 1 and a.task == "segmentation"
    assert a.cfg_options == {"runner.max_iters": 10, "model.decode_head.in_index": [3], "data.samples_per_gpu": 4}
    with pytest.raises(NotImplementedError, match="depth"):
        E.main(E.parse_args(["cfg.py", "--task", "depth"]))


@pytest.mark.parametrize("name", ["vitb_voc2012_linear_config.py", "vitb_ade20k_linear_config.py"])
def test_config_loader_reproduces_the_reference_configs(tmp_path, name):
    with open(os.path.join(GOLDEN, "dense_eval_configs.json")) as fh:
        gold = json.load(fh)[name]
    path = tmp_path / name
    path.write_text("".join(f"{k} = {v!r}\n" for k, v in gold.items()).replace("null", "None"))
    cfg = C.load_config(str(path))
    assert _jsonable(cfg) == gold
    C.check_supported(cfg)
    C.merge_options(cfg, {"runner.max_iters": 100, "model.decode_head.num_classes": 7, "data.train.pipeline.4.prob": 0.25,
                          "evaluation.interval": 50, "model.decode_head.in_channels": [384]})
    assert cfg["runner"]["max_iters"] == 100 and cfg["model"]["decode_head"]["num_classes"] == 7
    assert cfg["data"]["train"]["pipeline"][4] == {"type": "RandomFlip", "prob": 0.25}
    assert cfg["evaluation"] == {"interval": 50, "metric": "mIoU", "pre_eval": True}
    assert cfg["model"]["decode_head"]["in_channels"] == [384]


def test_cfg_option_values_parse_like_mmcv():
    assert C.parse_value("1") == 1 and C.parse_value("1e-3") == 1e-3 and C.parse_value("True") is True
    assert C.parse_value("None") is None and C.parse_value("abc") == "abc"
    assert C.parse_value("[1,2]") == [1, 2] and C.parse_value("1,2") == [1, 2]
    assert C.parse_value("[(1,2),(3,4)]") == [(1, 2), (3, 4)] and C.parse_value("'(512,512)'") == (512, 512)


def test_config_loader_refuses_what_it_does_not_implement(tmp_path):
    p = tmp_path / "base.py"
    p.write_text("_base_ = ['x.py']\n")
    with pytest.raises(C.ConfigError, match="_base_"):
        C.load_config(str(p))
    with open(os.path.join(GOLDEN, "dense_eval_configs.json")) as fh:
        gold = json.load(fh)["vitb_voc2012_linear_config.py"]
    for key, val, msg in [("model.decode_head.type", "UPerHead", "BNHead"),
                          ("data.train.pipeline.2.type", "RandomRotate", "RandomRotate"),
                          ("model.test_cfg.mode", "whole", "slide"),
                          ("lr_config.policy", "step", "poly")]:
        cfg = json.loads(json.dumps(gold))
        C.merge_options(cfg, {key: val})
        with pytest.raises(C.ConfigError, match=msg):
            C.check_supported(cfg)


def test_keep_ratio_resize_sizes():
    # (h, w) into (2048, 512): factor min(2048 / long, 512 / short), sizes rounded half up
    assert D.rescale_size(375, 500, (2048, 512)) == (512, 683)
    assert D.rescale_size(512, 2048, (2048, 512)) == (512, 2048)
    assert D.rescale_size(100, 1000, (2048, 512)) == (205, 2048)
    assert D.rescale_size(333, 500, (1024, 256)) == (256, 384)


@pytest.mark.parametrize("H, W, expect_rows, expect_cols", [
    (300, 200, [(0, 300)], [(0, 200)]),                                  # smaller than the crop
    (512, 512, [(0, 512)], [(0, 512)]),                                  # equal to the crop
    (512, 683, [(0, 512)], [(0, 512), (171, 683)]),                      # not a multiple of crop / stride
    (1000, 2048, [(0, 512), (341, 853), (488, 1000)],
     [(0, 512), (341, 853), (682, 1194), (1023, 1535), (1364, 1876), (1536, 2048)]),
])
def test_slide_window_grid(H, W, expect_rows, expect_cols):
    wins = D.slide_windows(H, W, (512, 512), (341, 341))
    assert wins == [(y1, y2, x1, x2) for (y1, y2) in expect_rows for (x1, x2) in expect_cols]


def test_pad_normalize_and_reduce_zero_label():
    img = np.arange(2 * 3 * 3, dtype=np.uint8).reshape(2, 3, 3)
    r = D.Normalize(mean=[1.0, 2.0, 3.0], std=[2.0, 4.0, 8.0], to_rgb=True)({"img": img}, None)
    np.testing.assert_allclose(r["img"][1, 2], [(15 - 1) / 2, (16 - 2) / 4, (17 - 3) / 8])
    r = D.Normalize(mean=[1.0, 2.0, 3.0], std=[2.0, 4.0, 8.0], to_rgb=False)({"img": img}, None)
    np.testing.assert_allclose(r["img"][0, 0], [(2 - 1) / 2, (1 - 2) / 4, (0 - 3) / 8])
    seg = np.array([[0, 1], [2, 255]], np.uint8)
    r = D.Pad(size=(3, 4), pad_val=0, seg_pad_val=255)({"img": np.ones((2, 2, 3), np.float32), "seg": seg}, None)
    assert r["img"].shape == (3, 4, 3) and r["img"][:2, :2].sum() == 12 and r["img"].sum() == 12
    assert (r["seg"] == np.array([[0, 1, 255, 255], [2, 255, 255, 255], [255] * 4])).all()
    assert (D.reduce_zero_label(np.array([0, 1, 2, 150, 255], np.uint8)) == [255, 0, 1, 149, 255]).all()


def _sample(h=300, w=400):
    yy, xx = np.mgrid[0:h, 0:w]
    img = np.stack([yy % 256, xx % 256, (yy // 256) * 16 + xx // 256], -1).astype(np.uint8)   # unique per pixel
    seg = ((yy // 50) * 3 + (xx // 100)).astype(np.uint8) % 5
    seg[:10] = 255
    return img, seg


def test_random_transforms_keep_image_and_label_aligned():
    img, seg = _sample()
    code = img[..., 0].astype(np.int64) * 65536 + img[..., 1].astype(np.int64) * 256 + img[..., 2]
    lut = {c: s for c, s in zip(code.ravel().tolist(), seg.ravel().tolist())}
    for seed in range(6):
        rng = np.random.RandomState(seed)
        r = {"img": img, "seg": seg}
        for t in (D.RandomCrop((128, 160), cat_max_ratio=0.75), D.RandomFlip(prob=0.5)):
            r = t(r, rng)
        assert r["img"].shape == (128, 160, 3) and r["seg"].shape == (128, 160)
        c = r["img"][..., 0].astype(np.int64) * 65536 + r["img"][..., 1].astype(np.int64) * 256 + r["img"][..., 2]
        assert all(lut[a] == b for a, b in zip(c.ravel().tolist(), r["seg"].ravel().tolist()))


def test_random_crop_respects_cat_max_ratio():
    seg = np.zeros((200, 200), np.uint8)
    seg[:, 150:] = 1                       # class 1 covers a quarter: most crops are dominated by class 0
    img = np.zeros((200, 200, 3), np.uint8)
    for seed in range(10):
        r = D.RandomCrop((100, 100), cat_max_ratio=0.75)({"img": img, "seg": seg}, np.random.RandomState(seed))
        _, cnt = np.unique(r["seg"], return_counts=True)
        assert len(cnt) > 1 and cnt.max() / cnt.sum() < 0.75


def test_resize_and_photometric_keep_shapes_and_are_seeded():
    img, seg = _sample()
    steps = [D.Resize(img_scale=(2048, 512), ratio_range=(0.5, 2.0)), D.RandomCrop((512, 512), cat_max_ratio=0.75),
             D.RandomFlip(prob=0.5), D.PhotoMetricDistortion(),
             D.Normalize(mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375]), D.Pad(size=(512, 512))]
    outs = []
    for _ in range(2):
        r, rng = {"img": img, "seg": seg}, np.random.RandomState(3)
        for t in steps:
            r = t(r, rng)
        outs.append(r)
    assert outs[0]["img"].shape == (512, 512, 3) and outs[0]["seg"].shape == (512, 512)
    assert np.array_equal(outs[0]["img"], outs[1]["img"]) and np.array_equal(outs[0]["seg"], outs[1]["seg"])


def test_hsv_round_trip():
    rgb = np.random.RandomState(0).randint(0, 256, (64, 64, 3)).astype(np.uint8)
    back = D.hsv2rgb(D.rgb2hsv(rgb)).astype(np.int64)
    assert np.abs(back - rgb).max() <= 4


@pytest.mark.parametrize("it", [0, 1, 1499, 1500, 39999])
def test_poly_lr_with_linear_warmup(it):
    base, max_iters, wi, ratio = 1e-3, 40000, 1500, 1e-6
    regular = base * (1 - it / max_iters)
    expect = regular * (1 - (1 - it / wi) * (1 - ratio)) if it < wi else regular
    got = poly_lr(it, base, max_iters, power=1.0, min_lr=0.0, warmup="linear", warmup_iters=wi, warmup_ratio=ratio)
    assert math.isclose(got, expect, rel_tol=1e-12, abs_tol=0)
    if it == 0:
        assert math.isclose(got, base * ratio, rel_tol=1e-9)


def test_metrics_from_histograms_match_numpy():
    rs = np.random.RandomState(0)
    K = 6
    pred = rs.randint(0, K - 1, 5000)            # class K-1 never predicted
    gt = rs.randint(0, K - 2, 5000)              # classes K-2, K-1 never in the ground truth
    gt[:300] = 255
    m = gt != 255
    p, g = pred[m], gt[m]
    inter = np.bincount(p[p == g], minlength=K)
    ap, al = np.bincount(p, minlength=K), np.bincount(g, minlength=K)
    hist = np.stack([inter, ap + al - inter, ap, al])
    res = metrics_from_hist(hist)
    with np.errstate(divide="ignore", invalid="ignore"):
        iou, acc = inter / (ap + al - inter), inter / al
    assert math.isclose(res["mIoU"], np.nanmean(iou)) and math.isclose(res["mAcc"], np.nanmean(acc))
    assert math.isclose(res["aAcc"], inter.sum() / al.sum())
    assert res["IoU"][K - 1] is None and res["Acc"][K - 2] is None and res["IoU"][K - 2] == 0.0
