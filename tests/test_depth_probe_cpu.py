"""NYU depth probe without a GPU: the config against the executed reference config, the refusals, the schedules, the
split file and the transforms against hand-computed values, the float64 oracle against losses and metrics computed by
the reference's own code (goldens), the argument checks of the dvt_depth_* entry points, and the per-image metric
gather over a gloo world of 2."""
import ctypes
import json
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)

from dvt.dense_eval import config as C  # noqa: E402
from dvt.dense_eval import depth as D  # noqa: E402
from dvt.dense_eval import depth_data as DD  # noqa: E402
from oracle import depth as OD  # noqa: E402


def _gold_cfg():
    with open(os.path.join(GOLDEN, "depth_config.json")) as fh:
        return json.load(fh)


def _jsonable(v):
    if isinstance(v, dict):
        return {k: _jsonable(x) for k, x in v.items()}
    if isinstance(v, (list, tuple, range)):
        return [_jsonable(x) for x in v]
    return v


def test_config_loads_like_the_reference_and_is_supported(tmp_path):
    gold = _gold_cfg()
    path = tmp_path / "vitb_nyu_linear_config.py"
    path.write_text("".join(f"{k} = {v!r}\n" for k, v in gold.items()).replace("null", "None"))
    cfg = C.load_config(str(path))
    assert _jsonable(cfg) == gold
    C.check_supported_depth(cfg)
    assert cfg["model"]["decode_head"]["channels"] == 1536 and cfg["model"]["decode_head"]["n_bins"] == 256
    with pytest.raises(C.ConfigError, match="EncoderDecoder"):
        C.check_supported(cfg)      # the segmentation probe refuses it


@pytest.mark.parametrize("key,val,msg", [
    ("model.decode_head.classify", False, "classify"),
    ("model.decode_head.bins_strategy", "SID", "SID"),
    ("model.decode_head.norm_strategy", "softmax", "norm_strategy"),
    ("model.decode_head.type", "DPTHead", "DPTHead"),
    ("model.test_cfg.mode", "slide", "whole"),
    ("model.decode_head.n_bins", 512, "n_bins"),
    ("model.backbone.output_cls_token", False, "output_cls_token"),
    ("model.type", "EncoderDecoder", "DepthEncoderDecoder"),
])
def test_depth_refusals_name_the_item(key, val, msg):
    cfg = json.loads(json.dumps(_gold_cfg()))
    C.merge_options(cfg, {key: val})
    with pytest.raises(C.ConfigError, match=msg):
        C.check_supported_depth(cfg)


def test_evaluate_depth_takes_the_reference_flags():
    import evaluate_dense_tasks as E
    import evaluate_depth as ED
    assert ED.parse_args is E.parse_args
    a = ED.parse_args(["cfg.py", "--launcher", "none", "--load-denoiser-from", "d.pth", "--deterministic"])
    assert a.load_denoiser_from == "d.pth" and a.deterministic and a.launcher == "none"


SCHED = dict(max_iters=38400, min_lr_ratio=1e-8, warmup="linear", warmup_iters=12800, warmup_ratio=0.001)


def _cos(base, target, f):
    return target + 0.5 * (base - target) * (1 + math.cos(math.pi * f))


@pytest.mark.parametrize("it", [0, 11519, 12799, 12800, 38399])
def test_cosine_lr_and_one_cycle_beta1(it):
    base, target = 0.005, 0.005 * 1e-8
    regular = _cos(base, target, it / 38400)
    want = regular * (1 - (1 - it / 12800) * 0.999) if it < 12800 else regular
    assert D.cosine_lr(it, base, **SCHED) == pytest.approx(want, rel=1e-12)
    beta1 = {0: 0.95, 11519: 0.85, 38399: 0.95}.get(it)
    if beta1 is None:   # second phase, from iteration 11519 (0.85) to 38399 (0.95)
        beta1 = _cos(0.85, 0.95, (it - 11519) / (38399 - 11519)) if it > 11519 else _cos(0.95, 0.85, it / 11519)
    assert D.one_cycle_momentum(it, 38400) == pytest.approx(beta1, abs=1e-12)
    if it == 0:
        assert D.cosine_lr(0, base, **SCHED) == pytest.approx(5e-6, rel=1e-9)


def test_paramwise_custom_keys_substring_rule():
    keys = {"pos_embed": {"decay_mult": 0.0}, "cls_token": {"decay_mult": 0.0}, "norm": {"decay_mult": 0.0},
            "backbone": {"lr_mult": 0.1}}
    p = [torch.nn.Parameter(torch.zeros(1)) for _ in range(4)]
    g = D.param_groups([("decode_head.conv_depth.weight", p[0]), ("decode_head.conv_depth.bias", p[1]),
                        ("decode_head.norm.weight", p[2]), ("backbone.norm.bias", p[3])], 0.005, 0.01, keys)
    assert [(x["lr"], x["weight_decay"]) for x in g[:2]] == [(0.005, 0.01), (0.005, 0.01)]   # the config's keys miss the head
    assert g[2]["weight_decay"] == 0.0 and g[2]["lr"] == 0.005
    assert g[3]["lr"] == pytest.approx(0.0005) and g[3]["weight_decay"] == 0.01    # longest key first: "backbone"


def test_split_parsing(tmp_path):
    (tmp_path / "split.txt").write_text("/b/rgb_2.jpg /b/depth_2.png 518.8\n/a/rgb_1.jpg None 518.8\n"
                                        "a/rgb_0.jpg /a/depth_0.png 518.8\n\n")
    pairs = DD.parse_split(str(tmp_path / "split.txt"), "root")
    assert pairs == [("root/a/rgb_0.jpg", "root/a/depth_0.png"), ("root/b/rgb_2.jpg", "root/b/depth_2.png")]


def test_nyu_crop_flip_crop_and_color_channel_mapping():
    img = np.arange(480 * 640 * 3, dtype=np.int64).reshape(480, 640, 3) % 251
    img = img.astype(np.uint8)
    depth = np.arange(480 * 640, dtype=np.float32).reshape(480, 640)
    r = DD.NYUCrop(depth=True)({"img": img, "depth": depth}, None)
    assert r["img"].shape == (427, 565, 3) and r["depth"][0, 0] == depth[45, 43] and r["depth"][-1, -1] == depth[471, 607]
    rng = np.random.RandomState(3)
    flip = rng.rand() < 0.5
    oh, ow = rng.randint(0, 427 - 416 + 1), rng.randint(0, 565 - 544 + 1)
    rng = np.random.RandomState(3)
    r = DD.RandomFlip(prob=0.5)(r, rng)
    r = DD.RandomCrop((416, 544))(r, rng)
    src = depth[45:472, 43:608][:, ::-1] if flip else depth[45:472, 43:608]
    np.testing.assert_array_equal(r["depth"], src[oh:oh + 416, ow:ow + 544])
    # ColorAug: draws rand, gamma, brightness, colors[3] (BGR order); RGB channel c takes colors[2 - c]
    x = np.full((2, 2, 3), 100, np.uint8)
    rng = np.random.RandomState(0)
    u = rng.rand()
    gamma, bright, colors = rng.uniform(0.9, 1.1), rng.uniform(0.75, 1.25), rng.uniform(0.9, 1.1, size=3)
    out = DD.ColorAug(prob=1.0, gamma_range=[0.9, 1.1], brightness_range=[0.75, 1.25],
                      color_range=[0.9, 1.1])({"img": x}, np.random.RandomState(0))["img"]
    assert u < 1.0
    for c in range(3):
        assert out[0, 0, c] == pytest.approx(min(100 ** gamma * bright * colors[2 - c], 255))


def test_random_rotate_draw_order_and_a_known_pixel():
    h, w = 7, 9
    img = np.random.RandomState(1).randint(0, 255, (h, w, 3)).astype(np.uint8)
    depth = np.arange(h * w, dtype=np.float32).reshape(h, w) + 1
    # not rotating still draws the angle: the next draw is the same either way
    rng = np.random.RandomState(5)
    DD.RandomRotate(prob=0.0, degree=2.5)({"img": img, "depth": depth}, rng)
    ref = np.random.RandomState(5)
    ref.rand(), ref.uniform(-2.5, 2.5)
    assert rng.rand() == ref.rand()
    # 90 degrees about the centre (4, 3) of a 7 x 9 map: mmcv.imrotate turns clockwise, dst (x, y) = src of
    # (cx + (y - cy), cy - (x - cx))
    out = DD.rotate_nearest(depth, 90.0)
    assert out[3, 4] == depth[3, 4]
    assert out[3, 5] == depth[2, 4]   # dst (x=5, y=3) <- src (x=4, y=2)
    assert out[0, 0] == 0             # outside the source: border 0
    rot = DD.rotate_bilinear(img, 90.0)
    np.testing.assert_array_equal(rot[3, 5], img[2, 4])


def test_oracle_losses_match_the_reference_goldens():
    g = np.load(os.path.join(GOLDEN, "depth_losses.npz"))
    for B in (1, 2, 3, 5):
        pred, gt = torch.from_numpy(g[f"b{B}_pred"]), torch.from_numpy(g[f"b{B}_gt"])
        assert OD.sig_loss(pred, gt, True).item() == pytest.approx(float(g[f"b{B}_sig_warm"]), rel=1e-12)
        assert OD.sig_loss(pred, gt, False).item() == pytest.approx(float(g[f"b{B}_sig"]), rel=1e-12)
        assert (0.5 * OD.gradient_loss(pred, gt)).item() == pytest.approx(float(g[f"b{B}_grad"]), rel=1e-12, abs=0)
    assert float(g["b2_grad"]) == 0.0 and float(g["b1_grad"]) == 0.0 and float(g["b3_grad"]) > 0
    pred = torch.from_numpy(g["invalid_pred"])
    assert np.isnan(float(g["invalid_sig"])) and np.isnan(OD.sig_loss(pred, torch.zeros_like(pred), False).item())
    assert np.isnan(float(g["invalid_grad"])) and np.isnan(OD.gradient_loss(pred, torch.zeros_like(pred)).item())


def test_masked_losses_match_the_oracle_on_cpu():
    """depth_ops' mask-multiplied SigLoss / GradientLoss (what runs on the GPU) against the boolean-indexed oracle."""
    from dvt.dense_eval import depth_ops as O
    g = np.load(os.path.join(GOLDEN, "depth_losses.npz"))
    for B in (1, 2, 3, 5):
        pred = torch.from_numpy(g[f"b{B}_pred"]).requires_grad_(True)
        gt = torch.from_numpy(g[f"b{B}_gt"])
        for warm in (True, False):
            assert O.sig_loss(pred, gt, warm).item() == pytest.approx(OD.sig_loss(pred, gt, warm).item(), rel=1e-12)
        lg = O.gradient_loss(pred, gt)
        assert lg.item() == pytest.approx(OD.gradient_loss(pred, gt).item(), rel=1e-12, abs=1e-15)
        (dg,) = torch.autograd.grad(lg, pred)
        if B <= 2:
            assert lg.item() == 0 and torch.count_nonzero(dg) == 0
    s = O.SigLossState(True, 2)
    p, t = torch.from_numpy(g["b2_pred"]), torch.from_numpy(g["b2_gt"])
    vals = [s(p, t).item() for _ in range(3)]
    assert vals[0] == vals[1] == pytest.approx(float(g["b2_sig_warm"])) and vals[2] == pytest.approx(float(g["b2_sig"]))


def test_oracle_metrics_and_sums_match_the_reference_goldens():
    g = np.load(os.path.join(GOLDEN, "depth_metrics.npz"))
    for i in range(3):
        gt, pred, want = g[f"m{i}_gt"], g[f"m{i}_pred"], g[f"m{i}_out"]
        got = OD.calculate(gt.astype(np.float64), pred.astype(np.float64))
        np.testing.assert_allclose(got, want, rtol=2e-5, atol=1e-3, equal_nan=True)
        # the kernel's f64 sums, formed on the host, give the same metrics
        gd, pd = gt.astype(np.float64), pred.astype(np.float64)
        ratio = np.maximum(gt / pred, pred / gt)
        d, err = gd - pd, np.log(pd) - np.log(gd)
        sums = [gt.size, (ratio < 1.25).sum(), (ratio < 1.25 ** 2).sum(), (ratio < 1.25 ** 3).sum(), (np.abs(d) / gd).sum(),
                (d * d / gd).sum(), (d * d).sum(), err.sum(), (err * err).sum(), np.abs(np.log10(gd) - np.log10(pd)).sum()]
        np.testing.assert_allclose(D.metrics_from_sums(sums), want, rtol=2e-5, atol=1e-3, equal_nan=True)
    assert np.isnan(D.metrics_from_sums([0] * 10)).all()
    assert D.summarize(np.array([[np.nan] * 9, [1.0] * 9]))["abs_rel"] == 1.0


def test_depth_entry_points_reject_bad_arguments():
    from dvt import _lib
    L = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    cases = [
        (L.dvt_depth_head_fwd, (None, 1, 2, 2, 8, 4, p, p, None), "null"),
        (L.dvt_depth_head_fwd, (p, 1, 2, 2, 300, 4, p, p, None), "n_bins"),
        (L.dvt_depth_head_fwd, (p, 0, 2, 2, 8, 4, p, p, None), "bad shape"),
        (L.dvt_depth_head_bwd, (p, 1, 2, 2, 8, 4, p, None, p, None), "null"),
        (L.dvt_depth_head_bwd, (p, 1, 2, 2, 8, 0, p, p, p, None), "bad shape"),
        (L.dvt_depth_resize_fwd, (p, 1, 0, 2, p, 4, 4, None), "bad shape"),
        (L.dvt_depth_resize_bwd, (None, 1, 2, 2, 4, 4, p, None), "null"),
        (L.dvt_depth_eval_sums, (p, 0, 0, 2, 2, p, 4, 4, 0.001, 10.0, 0, 4, 0, 4, p, p, None), "n_aug"),
        (L.dvt_depth_eval_sums, (p, 1, 0, 2, 2, p, 4, 4, 10.0, 1.0, 0, 4, 0, 4, p, p, None), "min_depth"),
        (L.dvt_depth_eval_sums, (p, 1, 0, 2, 2, None, 4, 4, 0.001, 10.0, 0, 4, 0, 4, p, p, None), "null"),
    ]
    for fn, args, msg in cases:
        assert fn(*args) != 0
        assert msg in L.dvt_last_error().decode()


def _gather_worker(rank, world, init):
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=init, rank=rank, world_size=world)
    n = 5
    mine = list(range(rank, n, world))
    rows = np.array([[float(i)] * 9 for i in mine])
    out = D.gather_rows(mine, rows, n)
    assert np.array_equal(out[:, 0], np.arange(n, dtype=np.float64))
    assert D.summarize(out)["rmse"] == 2.0
    dist.destroy_process_group()


def test_metric_rows_gather_over_two_ranks(tmp_path):
    import torch.multiprocessing as mp
    mp.spawn(_gather_worker, args=(2, f"file://{tmp_path}/store"), nprocs=2, join=True)
