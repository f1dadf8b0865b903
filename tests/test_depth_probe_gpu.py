"""NYU depth probe on the GPU: the bin-expectation head kernel, the one-channel resize and the fused evaluation against
the float64 restatement (oracle/depth.py) and the reference-minted metrics, the probe's features plus cls against
get_intermediate_layers, and evaluate_depth.py end to end on a synthetic NYU-layout set."""
import glob
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)

from oracle import depth as OD  # noqa: E402

pytestmark = pytest.mark.gpu


def _head_case(B, h, w, K, C=48, H=None, W=None, seed=0):
    g = torch.Generator().manual_seed(seed * 1000 + B * 100 + h + K)
    feat = torch.randn(B, h, w, C, generator=g)
    cls = torch.randn(B, C, generator=g)
    conv = torch.nn.Conv2d(2 * C, K, 1)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(K, 2 * C, 1, 1, generator=g) * 0.3)
        conv.bias.copy_(torch.randn(K, generator=g) * 0.1)
    H, W = H or 14 * h - 4, W or 14 * w - 2
    gt = torch.rand(B, H, W, generator=g) * 9 + 0.5
    gt[torch.rand(B, H, W, generator=g) < 0.1] = 0
    return feat, cls, conv, gt


@pytest.mark.parametrize("h, w", [(30, 39), (35, 46), (7, 9)])
@pytest.mark.parametrize("B", [1, 2, 3])
@pytest.mark.parametrize("K", [256, 100])
def test_head_loss_and_weight_gradients_match_float64(h, w, B, K):
    from dvt.dense_eval import depth_ops as O
    from dvt.dense_eval.depth import DepthHead, depth_losses
    feat, cls, conv, gt = _head_case(B, h, w, K)
    # float64 oracle: upsample the features, conv, relu, normalise, einsum, resize, SigLoss + GradientLoss
    w64 = conv.weight.detach().double().requires_grad_(True)
    b64 = conv.bias.detach().double().requires_grad_(True)
    bins64 = torch.linspace(0.001, 10, K, dtype=torch.float64)
    d4 = OD.head_forward(feat.double().permute(0, 3, 1, 2), cls.double(), w64, b64, bins64, 4)
    ld, lg, tot = OD.loss(d4, gt.double()[:, None], warm_up=False)
    tot.backward()
    torch.use_deterministic_algorithms(True)
    try:
        outs = []
        for _ in range(3):
            head = DepthHead(2 * feat.shape[-1], K, 0.001, 10, 4).cuda()
            head.conv_depth.load_state_dict(conv.state_dict())
            sig = O.SigLossState(warm_up=False)
            losses = depth_losses(head(feat.cuda(), cls.cuda()), gt.cuda(), sig, 1.0, 0.5)
            losses["loss"].backward()
            outs.append((losses["loss"].detach().cpu(), head.conv_depth.weight.grad.cpu(), head.conv_depth.bias.grad.cpu()))
    finally:
        torch.use_deterministic_algorithms(False)
    loss, dw, db = outs[0]
    assert loss.item() == pytest.approx(tot.item(), rel=1e-5)
    assert losses["decode.loss_grad"].item() == pytest.approx(lg.item(), rel=1e-5, abs=1e-7)
    if B <= 2:
        assert losses["decode.loss_grad"].item() == 0
    # dW / db: the kernel's low-resolution gradient (checked alone below) goes through fp32 cuBLAS GEMMs and loss
    # reductions whose sums cancel over the image; norm-wise relative error
    assert ((dw.double() - w64.grad).norm() / w64.grad.norm()).item() < 1e-4
    assert ((db.double() - b64.grad).norm() / b64.grad.norm()).item() < 1e-4
    for o in outs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(outs[0], o))


@pytest.mark.parametrize("B", [1, 2, 3])
@pytest.mark.parametrize("K", [256, 100])
def test_head_kernel_gradient_matches_float64(B, K):
    from dvt.dense_eval import depth_ops as O
    feat, cls, conv, _ = _head_case(B, 35, 46, K)
    lg = O.head_logits(feat.cuda(), cls.cuda(), conv.weight.detach().cuda(), conv.bias.detach().cuda()).detach()
    bins = torch.linspace(0.001, 10, K, device="cuda")
    x = lg.clone().requires_grad_(True)
    d4 = O.bin_expectation(x, bins, 4)
    gd = torch.randn(d4.shape, generator=torch.Generator().manual_seed(B)).cuda()
    d4.backward(gd)
    x64 = lg.double().cpu().requires_grad_(True)
    up = F.interpolate(x64.permute(0, 3, 1, 2), size=(140, 184), mode="bilinear", align_corners=False)
    a = torch.relu(up) + 0.1
    r = torch.einsum("ikmn,k->imn", a / a.sum(1, keepdim=True), bins.double().cpu())
    r.backward(gd.double().cpu())
    assert ((d4.double().cpu() - r).abs().max() / r.abs().max()).item() < 1e-5
    assert ((x.grad.double().cpu() - x64.grad).abs().max() / x64.grad.abs().max()).item() < 1e-5


@pytest.mark.parametrize("Hi, Wi, Ho, Wo", [(120, 156, 416, 544), (140, 184, 480, 640), (9, 7, 5, 11)])
def test_resize_matches_interpolate_and_float64_autograd(Hi, Wi, Ho, Wo):
    from dvt.dense_eval import depth_ops as O
    g = torch.Generator().manual_seed(Hi + Wo)
    x = torch.randn(2, Hi, Wi, generator=g)
    dout = torch.randn(2, Ho, Wo, generator=g)
    xc = x.cuda().requires_grad_(True)
    out = O.resize(xc, (Ho, Wo))
    ref = F.interpolate(x.cuda()[:, None], size=(Ho, Wo), mode="bilinear", align_corners=False)[:, 0]
    assert (out - ref).abs().max().item() <= 1e-6 * ref.abs().max().item()
    out.backward(dout.cuda())
    # against ATen's own fp32 backward (same fp32 tap weights, scattered): 1e-5; against float64 autograd, whose tap
    # weights come from float64 source indices (up to ~5e-6 apart at 640 pixels), 1e-4
    x32 = x.cuda().requires_grad_(True)
    F.interpolate(x32[:, None], size=(Ho, Wo), mode="bilinear", align_corners=False)[:, 0].backward(dout.cuda())
    scale = x32.grad.abs().max().item()
    assert (xc.grad - x32.grad).abs().max().item() < 1e-5 * scale
    x64 = x.double().requires_grad_(True)
    F.interpolate(x64[:, None], size=(Ho, Wo), mode="bilinear", align_corners=False)[:, 0].backward(dout.double())
    assert (xc.grad.cpu().double() - x64.grad).abs().max().item() < 1e-4 * scale
    torch.use_deterministic_algorithms(True)
    try:
        g2 = torch.autograd.grad(O.resize(xc, (Ho, Wo)), xc, dout.cuda())[0]
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.equal(g2, xc.grad)


@pytest.mark.parametrize("flip", [True, False])
def test_eval_sums_match_the_float64_restatement(flip):
    from dvt.dense_eval import depth_ops as O
    from dvt.dense_eval.depth import metrics_from_sums
    g = torch.Generator().manual_seed(7)
    Ho, Wo, Hu, Wu = 480, 640, 140, 184
    flips = [False, True] if flip else [False]
    maps = torch.rand(len(flips), Hu, Wu, generator=g) * 12 - 1       # outside [min, max] too: the clamp matters
    gt = torch.rand(Ho, Wo, generator=g) * 11
    gt[torch.rand(Ho, Wo, generator=g) < 0.2] = 0
    crop = (45, 471, 41, 601)
    out = torch.zeros(10, dtype=torch.float64, device="cuda")
    ws = torch.empty(O.EVAL_WORKSPACE, dtype=torch.float64, device="cuda")
    O.eval_sums(maps.cuda(), flips, gt.cuda(), 0.001, 10, crop, out, ws)
    got = metrics_from_sums(out.cpu().numpy())
    want = OD.image_metrics(maps[:, None].numpy(), flips, gt.numpy(), 0.001, 10, crop)
    np.testing.assert_allclose(got[[0, 1, 2]], want[[0, 1, 2]], atol=2e-5)
    np.testing.assert_allclose(got[3:], want[3:], rtol=1e-5, atol=1e-6)
    out2 = torch.zeros_like(out)
    O.eval_sums(maps.cuda(), flips, gt.cuda(), 0.001, 10, crop, out2, ws)
    assert torch.equal(out, out2)
    # every pixel invalid: an empty mask gives NaN
    O.eval_sums(maps.cuda(), flips, torch.zeros(Ho, Wo, device="cuda"), 0.001, 10, crop, out, ws)
    assert out[0].item() == 0 and np.isnan(metrics_from_sums(out.cpu().numpy())).all()


def test_eval_sums_match_the_reference_metrics():
    """calculate() of the reference on float32 gt / pred vectors (golden) against the kernel, with the prediction laid out
    as a 1-augmentation map of the image's own size (the resize is then the identity)."""
    from dvt.dense_eval import depth_ops as O
    from dvt.dense_eval.depth import metrics_from_sums
    gm = np.load(os.path.join(GOLDEN, "depth_metrics.npz"))
    for i in range(3):
        gt, pred, want = gm[f"m{i}_gt"], gm[f"m{i}_pred"], gm[f"m{i}_out"]
        n = max(gt.size, 1)
        gt_t = torch.zeros(1, n) if gt.size == 0 else torch.from_numpy(gt)[None]
        pred_t = torch.ones(1, 1, n) if pred.size == 0 else torch.from_numpy(pred)[None, None]
        out = torch.zeros(10, dtype=torch.float64, device="cuda")
        ws = torch.empty(O.EVAL_WORKSPACE, dtype=torch.float64, device="cuda")
        # max_depth 100: neither the clamp nor the mask binds, as in calculate() on the bare vectors
        O.eval_sums(pred_t.cuda(), [False], gt_t.cuda(), 0.001, 100, (0, 1, 0, n), out, ws)
        got = metrics_from_sums(out.cpu().numpy())
        if gt.size == 0:
            assert np.isnan(got).all() and np.isnan(want).all()
            continue
        np.testing.assert_allclose(np.delete(got, 7), np.delete(want, 7), rtol=1e-5, atol=1e-6)
        assert abs(got[7] - want[7]) < 1e-3


IDENT = "vit_small_patch14_dinov2.lvd142m"


@pytest.mark.parametrize("kind", ["plain", "reg4", "denoiser"])
def test_probe_features_and_cls_equal_get_intermediate_layers(kind):
    import dvt.models as DVT
    from dvt.dense_eval.model import ProbeBackbone
    ident = "vit_small_patch14_reg4_dinov2.lvd142m" if kind == "reg4" else IDENT
    torch.manual_seed(0)
    vit = DVT.PretrainedViTWrapper(ident, stride=14, allow_random_init=True).cuda().eval()
    x = torch.randn(2, 3, 416, 544).cuda()
    xp = F.pad(x, (1, 1, 2, 2))
    if kind == "denoiser":
        den = DVT.Denoiser(37, 37, 384, vit=vit, num_blocks=1).cuda().eval()
        probe = ProbeBackbone(den, [11], [0], return_cls=True, norm=True)
        feat, cls = probe(x)
        ref_f, ref_c = den(xp, return_class_token=True, norm=True)
        assert torch.equal(cls, ref_c)
        assert (feat - ref_f).abs().max().item() <= 1e-3 * ref_f.abs().max().item()
        return
    probe = ProbeBackbone(vit, [11], [0], return_cls=True, norm=True)
    feat, cls = probe(x)
    (ref,) = vit.get_intermediate_layers(xp, n=[11], reshape=True, return_prefix_tokens=True, norm=True)
    assert feat.shape == (2, 30, 39, 384) and cls.shape == (2, 384)
    assert torch.equal(feat, ref[0].permute(0, 2, 3, 1)) and torch.equal(cls, ref[1][:, 0])
    assert ref[1].shape[1] == (5 if kind == "reg4" else 1)


# ---------------------------------------------------------------------------------------------------------------------
# command line, end to end
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def nyu(tmp_path_factory):
    """NYU layout: 480 x 640 RGB JPEG-free PNGs and uint16 depth PNGs (millimetres), depth a smooth ramp plus the image's
    brightness, some pixels 0 (invalid); split lines `rgb depth focal`, one with depth None."""
    from PIL import Image
    root = tmp_path_factory.mktemp("nyu")
    rs = np.random.RandomState(0)
    lines = {"train": [], "test": []}
    for i in range(8):
        split = "train" if i < 6 else "test"
        d = root / split / f"scene{i}"
        d.mkdir(parents=True)
        yy, xx = np.mgrid[0:480, 0:640]
        depth = 1.0 + 6.0 * (yy / 480) + 2.0 * np.sin(xx / 80.0 + i)
        img = np.stack([depth * 30, 255 - depth * 25, (xx % 255)], -1) + rs.normal(0, 8, (480, 640, 3))
        Image.fromarray(np.clip(img, 0, 255).astype(np.uint8)).save(d / "rgb_00000.png")
        mm = (depth * 1000).astype(np.uint16)
        mm[rs.rand(480, 640) < 0.05] = 0
        Image.fromarray(mm).save(d / "sync_depth_00000.png")
        lines[split].append(f"/{split}/scene{i}/rgb_00000.png /{split}/scene{i}/sync_depth_00000.png 518.8579")
    lines["train"].append("/train/missing/rgb_00000.png None 518.8579")
    (root / "nyu_train.txt").write_text("\n".join(lines["train"]) + "\n")
    (root / "nyu_test.txt").write_text("\n".join(lines["test"]) + "\n")
    with open(os.path.join(GOLDEN, "depth_config.json")) as fh:
        gold = json.load(fh)
    (root / "nyu_linear.py").write_text("".join(f"{k} = {v!r}\n" for k, v in gold.items()).replace("null", "None"))
    return root


def _argv(nyu, work, iters, ckpt, evaluate, extra=()):
    return [str(nyu / "nyu_linear.py"), "--work-dir", str(work), "--launcher", "none", "--seed", "0",
            "--backbone-type", IDENT, "--cfg-options", f"data.train.data_root={nyu}", f"data.val.data_root={nyu}",
            "model.decode_head.in_channels=[384]", "model.decode_head.channels=768", f"runner.max_iters={iters}",
            f"checkpoint_config.interval={ckpt}", f"evaluation.interval={evaluate}", "log_config.interval=5",
            "lr_config.warmup_iters=10", "data.workers_per_gpu=2", *extra]


def _run(argv, monkeypatch):
    import evaluate_depth as ED
    monkeypatch.setenv("DVT_ALLOW_RANDOM_INIT", "1")
    monkeypatch.delenv("DVT_WEIGHTS_DIR", raising=False)
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    try:
        return ED.main(ED.parse_args(argv))
    finally:
        torch.use_deterministic_algorithms(False)


def _records(work):
    (log,) = glob.glob(str(work / "*.log.json"))
    return [json.loads(ln) for ln in open(log)]


def test_cli_trains_checkpoints_keeps_two_and_saves_the_best(nyu, tmp_path, monkeypatch):
    work = tmp_path / "work"
    out = _run(_argv(nyu, work, 40, ckpt=10, evaluate=10), monkeypatch)
    files = set(os.listdir(work))
    assert {"iter_30.pth", "iter_40.pth", "latest.pth"} <= files and "iter_10.pth" not in files and "iter_20.pth" not in files
    assert os.readlink(work / "latest.pth") == "iter_40.pth"
    best = [f for f in files if f.startswith("best_abs_rel_iter_")]
    assert len(best) == 1, files
    ck = torch.load(work / "latest.pth", map_location="cpu")
    assert set(ck["state_dict"]) == {"decode_head.conv_depth.weight", "decode_head.conv_depth.bias"}
    assert ck["state_dict"]["decode_head.conv_depth.weight"].shape == (256, 768, 1, 1)
    recs = _records(work)
    val = [r for r in recs if r.get("mode") == "val"]
    assert len(val) == 4 and all(np.isfinite(v[k]) for v in val for k in ("a1", "a2", "a3", "abs_rel", "rmse", "log_10",
                                                                            "rmse_log", "silog", "sq_rel"))
    best_iter = int(best[0].split("_")[-1][:-4])
    assert min(val, key=lambda v: v["abs_rel"])["iter"] == best_iter
    train = [r for r in recs if r.get("mode") == "train"]
    assert all({"decode.loss_depth", "decode.loss_grad", "loss"} <= set(r) for r in train)
    assert all(r["decode.loss_grad"] == 0 for r in train)       # batch 2: the reference's GradientLoss is 0
    assert out["sig_loss_calls"] == 40


def test_cli_deterministic_runs_are_bit_identical(nyu, tmp_path, monkeypatch):
    heads, logs = [], []
    for run in range(2):
        work = tmp_path / f"det{run}"
        _run(_argv(nyu, work, 15, ckpt=15, evaluate=15, extra=("--deterministic",)), monkeypatch)
        heads.append(torch.load(work / "latest.pth", map_location="cpu")["state_dict"])
        logs.append([{k: v for k, v in r.items()} for r in _records(work) if r.get("mode") in ("train", "val")])
    assert all(torch.equal(heads[0][k], heads[1][k]) for k in heads[0])
    assert logs[0] == logs[1]


def test_cli_resume_warms_sigloss_up_again_and_other_backbones(nyu, tmp_path, monkeypatch):
    import dvt.models as DVT
    work = tmp_path / "work"
    _run(_argv(nyu, work, 10, ckpt=5, evaluate=100, extra=("--no-validate",)), monkeypatch)
    out = _run(_argv(nyu, work, 15, ckpt=5, evaluate=100,
                     extra=("--no-validate", "--resume-from", str(work / "iter_5.pth"))), monkeypatch)
    assert out["sig_loss_calls"] == 10           # iterations 5..14 of the resumed run, counted from 0 again
    assert torch.load(work / "latest.pth", map_location="cpu")["iter"] == 15
    torch.manual_seed(1)
    den = DVT.Denoiser(37, 37, 384, vit=None, num_blocks=1)
    torch.save({"denoiser": den.state_dict()}, tmp_path / "denoiser.pth")
    vit = DVT.PretrainedViTWrapper(IDENT, stride=14, allow_random_init=True)
    torch.save({"model": vit.state_dict()}, tmp_path / "distilled.pth")
    for flag, path in (("--load-denoiser-from", "denoiser.pth"), ("--load-distilled-model-from", "distilled.pth")):
        w = tmp_path / flag.strip("-")
        _run(_argv(nyu, w, 6, ckpt=6, evaluate=6, extra=(flag, str(tmp_path / path))), monkeypatch)
        val = [r for r in _records(w) if r.get("mode") == "val"]
        assert len(val) == 1 and np.isfinite(val[0]["abs_rel"])
