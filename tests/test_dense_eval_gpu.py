"""Segmentation probe on the GPU: the fused upsample + cross-entropy kernel against the float64 torch statement under
autograd, slide inference against a torch restatement of mmseg's slide_inference, the probe's backbone features against
the wrapper, and evaluate_dense_tasks.py end to end on a synthetic VOC-layout dataset (plain, denoised and distilled
backbones, resume, and two --deterministic runs)."""
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

pytestmark = pytest.mark.gpu


def _labels(B, H, W, K, seed, ignore_frac=0.05, all_ignored=()):
    g = torch.Generator().manual_seed(seed)
    lab = torch.randint(0, K, (B, H, W), generator=g, dtype=torch.int64)
    lab[torch.rand(B, H, W, generator=g) < ignore_frac] = 255
    for b in all_ignored:
        lab[b] = 255
    return lab.to(torch.uint8).cuda()


@pytest.mark.parametrize("K", [21, 150])
@pytest.mark.parametrize("h, w, H, W", [(37, 37, 512, 512), (37, 37, 500, 375), (32, 32, 512, 512)])
@pytest.mark.parametrize("all_ignored", [False, True])
def test_upsample_ce_matches_float64_autograd(K, h, w, H, W, all_ignored):
    from dvt.dense_eval import seg_ops
    B = 2
    g = torch.Generator().manual_seed(K * 1000 + h + H)
    logits = (torch.randn(B, h, w, K, generator=g) * 3).cuda()
    labels = _labels(B, H, W, K, seed=H + W, all_ignored=(1,) if all_ignored else ())
    ref_in = logits.double().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    up = F.interpolate(ref_in, size=(H, W), mode="bilinear", align_corners=False)
    ref = F.cross_entropy(up, labels.long(), reduction="none", ignore_index=255).mean()
    ref.backward()
    ref_grad = ref_in.grad.permute(0, 2, 3, 1)
    x = logits.clone().requires_grad_(True)
    loss = seg_ops.upsample_cross_entropy(x, labels)
    loss.backward()
    assert abs(loss.item() - ref.item()) <= 1e-5 * abs(ref.item())
    err = (x.grad.double() - ref_grad).norm() / ref_grad.norm()
    assert err <= 1e-5, err.item()
    assert (x.grad.double() - ref_grad).abs().max() <= 1e-5 * ref_grad.abs().max()
    if all_ignored:
        assert torch.count_nonzero(x.grad[1]) == 0
    outs = [seg_ops.upsample_ce_sum(logits, labels, 1.0 / labels.numel()) for _ in range(3)]
    for l2, d2 in outs[1:]:
        assert torch.equal(l2, outs[0][0]) and torch.equal(d2, outs[0][1])
    assert torch.equal(outs[0][1], x.grad)


def _mmseg_slide_torch(logits_fn, img, crop, stride, K, out_size):
    """mmseg 0.27 EncoderDecoder.slide_inference + the rescale of `inference`, restated in torch (fp32)."""
    from dvt.dense_eval.data import slide_windows
    H, W = img.shape[1:]
    preds = torch.zeros(1, K, H, W, device=img.device)
    count = torch.zeros(1, 1, H, W, device=img.device)
    for (y1, y2, x1, x2) in slide_windows(H, W, crop, stride):
        crop_logit = logits_fn(img[None, :, y1:y2, x1:x2]).permute(0, 3, 1, 2)
        crop_logit = F.interpolate(crop_logit, size=(y2 - y1, x2 - x1), mode="bilinear", align_corners=False)
        preds += F.pad(crop_logit, (x1, W - x2, y1, H - y2))
        count[:, :, y1:y2, x1:x2] += 1
    preds = preds / count
    return F.interpolate(preds, size=out_size, mode="bilinear", align_corners=False)[0]


def _hist_np(pred, gt, K):
    m = gt != 255
    p, g = pred[m], gt[m]
    inter = np.bincount(p[p == g], minlength=K)[:K]
    ap = np.bincount(p, minlength=K)[:K]
    al = np.bincount(g[g < K], minlength=K)[:K]
    return np.stack([inter, ap + al - inter, ap, al])


@pytest.mark.parametrize("K", [21, 150])
@pytest.mark.parametrize("H, W", [(300, 200), (512, 512), (512, 683), (1000, 2048)])
def test_slide_inference_matches_torch_restatement(K, H, W):
    from dvt.dense_eval import seg_ops
    from dvt.models import CenterPadding
    g = torch.Generator().manual_seed(K + H + W)
    w1 = (torch.randn(32, 3, 14, 14, generator=g) * 0.1).cuda()
    w2 = torch.randn(K, 32, generator=g).cuda()
    pad = CenterPadding(14)

    def logits_fn(crops):                                    # a random "backbone + head": NHWC logits at patch resolution
        f = torch.tanh(F.conv2d(pad(crops), w1, stride=14)).permute(0, 2, 3, 1)
        return f @ w2.t()

    img = torch.randn(3, H, W, generator=g).cuda()
    Ho, Wo = H * 3 // 4 + 1, W * 3 // 4 + 3
    gt = _labels(1, Ho, Wo, K, seed=7)[0]
    ref = _mmseg_slide_torch(logits_fn, img, (512, 512), (341, 341), K, (Ho, Wo))
    top2 = ref.topk(2, dim=0).values
    ties = ((top2[0] - top2[1]).abs() <= 1e-5 * top2[0].abs().clamp_min(1.0)) & (gt != 255)
    ref_hist = _hist_np(ref.argmax(0).cpu().numpy(), gt.cpu().numpy(), K)
    hist = torch.zeros(4, K, dtype=torch.int64, device="cuda")
    seg_ops.slide_inference_hist(logits_fn, img, gt, K, (512, 512), (341, 341), hist, max_batch=4)
    diff = np.abs(hist.cpu().numpy() - ref_hist)
    n_ties = int(ties.sum())
    assert diff.sum() <= 6 * n_ties, (diff.sum(), n_ties)     # one pixel moves at most 1 + 2 + 2 + 0 histogram counts
    assert hist[3].sum().item() == int(((gt != 255) & (gt < K)).sum())
    assert hist[2].sum().item() == int((gt != 255).sum())


def test_probe_features_equal_get_intermediate_layers():
    import dvt.models as DVT
    from dvt.dense_eval.model import ProbeBackbone
    from oracle import vit as OV
    cfg = OV.CONFIGS["vit_small_patch14_dinov2.lvd142m"]
    sd = OV.random_state_dict(cfg, seed=0)                   # LayerScale U(0.5, 1.5): the blocks matter
    vit = DVT.PretrainedViTWrapper("vit_small_patch14_dinov2.lvd142m", stride=14, allow_random_init=True)
    vit.model.load_state_dict(sd)
    vit = vit.cuda().eval()
    probe = ProbeBackbone(vit, [8, 9, 10, 11], [3])
    assert probe.layers == [11] and probe.channels == 384
    x = torch.randn(2, 3, 512, 512).cuda()
    got = probe(x)
    xp = F.pad(x, (3, 3, 3, 3))
    # the reference binds timm's get_intermediate_layers, whose norm defaults to False: no final LayerNorm
    ref = vit.get_intermediate_layers(xp, n=[11], reshape=True, norm=False)[0].permute(0, 2, 3, 1)
    assert got.shape == (2, 37, 37, 384) and torch.equal(got, ref)
    all4 = vit.get_intermediate_layers(xp, n=[8, 9, 10, 11], reshape=True, norm=False)
    assert torch.equal(all4[3].permute(0, 2, 3, 1), got)
    normed = vit.get_intermediate_layers(xp, n=[11], reshape=True, norm=True)[0].permute(0, 2, 3, 1)
    assert (normed - got).abs().max() > 1e-2
    # the un-normalised map is the oracle's block-11 output without the final norm
    oref = OV.forward_intermediates(sd, cfg, xp[:1].cpu(), [11], stride=14, norm=False)[0].permute(0, 2, 3, 1)
    cos = F.cosine_similarity(got[:1].cpu().reshape(-1, 384), oref.reshape(-1, 384), dim=-1).min()
    assert cos > 0.999, cos.item()


# ---------------------------------------------------------------------------------------------------------------------
# command line, end to end
# ---------------------------------------------------------------------------------------------------------------------
COLOURS = {0: (110, 110, 110), 1: (200, 40, 40), 2: (40, 190, 60), 3: (50, 60, 210)}
IDENT = "vit_small_patch14_dinov2.lvd142m"


def _palette_png(seg, path):
    from PIL import Image
    im = Image.fromarray(seg, mode="P")
    pal = [0] * 768
    for c, rgb in COLOURS.items():
        pal[3 * c:3 * c + 3] = rgb
    im.putpalette(pal)
    im.save(path)


@pytest.fixture(scope="module")
def voc(tmp_path_factory):
    """VOC layout: 3 coloured rectangles (classes 1-3, the label is the colour) on a grey background (class 0), noise on
    the pixels, the rectangles' borders ignored (255)."""
    from PIL import Image
    root = tmp_path_factory.mktemp("voc")
    for d in ("JPEGImages", "SegmentationClass", "ImageSets/Segmentation"):
        (root / d).mkdir(parents=True)
    rs = np.random.RandomState(0)
    names = []
    for i in range(20):
        H, W = rs.randint(220, 300), rs.randint(260, 360)
        img = np.zeros((H, W, 3), np.float32) + COLOURS[0]
        seg = np.zeros((H, W), np.uint8)
        for c in (1, 2, 3):
            h, w = rs.randint(50, 120), rs.randint(50, 120)
            y, x = rs.randint(0, H - h), rs.randint(0, W - w)
            img[y:y + h, x:x + w] = COLOURS[c]
            seg[y:y + h, x:x + w] = c
            seg[y:y + h, x] = 255
        img = np.clip(img + rs.normal(0, 12, img.shape), 0, 255).astype(np.uint8)
        name = f"img{i:03d}"
        Image.fromarray(img).save(root / "JPEGImages" / f"{name}.jpg", quality=95)
        _palette_png(seg, root / "SegmentationClass" / f"{name}.png")
        names.append(name)
    (root / "ImageSets/Segmentation/train.txt").write_text("\n".join(names[:16]) + "\n")
    (root / "ImageSets/Segmentation/val.txt").write_text("\n".join(names[16:]) + "\n")
    with open(os.path.join(GOLDEN, "dense_eval_configs.json")) as fh:
        gold = json.load(fh)["vitb_voc2012_linear_config.py"]
    cfg = root / "voc_linear.py"
    cfg.write_text("".join(f"{k} = {v!r}\n" for k, v in gold.items()).replace("null", "None"))
    return root


def _argv(voc, work, iters, extra=(), ckpt=None, evaluate=None):
    return [str(voc / "voc_linear.py"), "--work-dir", str(work), "--launcher", "none", "--seed", "0",
            "--backbone-type", IDENT, "--cfg-options", f"data_root={voc}", f"data.train.data_root={voc}",
            f"data.val.data_root={voc}", "model.decode_head.num_classes=4", "model.decode_head.in_channels=[384]",
            "model.decode_head.channels=384", f"runner.max_iters={iters}", f"checkpoint_config.interval={ckpt or iters}",
            f"evaluation.interval={evaluate or iters}", "log_config.interval=10", "lr_config.warmup_iters=10",
            "data.samples_per_gpu=4", "data.workers_per_gpu=2", *extra]


def _run(argv, monkeypatch):
    sys.path.insert(0, ROOT)
    import evaluate_dense_tasks as E
    monkeypatch.setenv("DVT_ALLOW_RANDOM_INIT", "1")
    monkeypatch.delenv("DVT_WEIGHTS_DIR", raising=False)
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    try:
        return E.main(E.parse_args(argv))
    finally:
        torch.use_deterministic_algorithms(False)


def _val_records(work):
    (log,) = glob.glob(str(work / "*.log.json"))
    recs = [json.loads(ln) for ln in open(log)]
    return recs, [r for r in recs if r.get("mode") == "val"]


def test_cli_trains_checkpoints_and_beats_chance(voc, tmp_path, monkeypatch):
    work = tmp_path / "work"
    _run(_argv(voc, work, 200, ckpt=100), monkeypatch)
    assert {"iter_100.pth", "iter_200.pth", "latest.pth"} <= set(os.listdir(work))
    assert os.readlink(work / "latest.pth") == "iter_200.pth"
    ck = torch.load(work / "latest.pth", map_location="cpu")
    assert set(ck) >= {"state_dict", "optimizer", "iter"} and ck["iter"] == 200
    assert set(ck["state_dict"]) == {"decode_head.bn.weight", "decode_head.bn.bias", "decode_head.bn.running_mean",
                                     "decode_head.bn.running_var", "decode_head.bn.num_batches_tracked",
                                     "decode_head.conv_seg.weight", "decode_head.conv_seg.bias"}
    assert ck["state_dict"]["decode_head.conv_seg.weight"].shape == (4, 384, 1, 1)
    recs, val = _val_records(work)
    train = [r["loss"] for r in recs if r.get("mode") == "train"]
    assert len(train) == 20 and train[-1] < 0.5 * train[0], train
    assert len(val) == 1 and val[0]["iter"] == 200 and len(val[0]["IoU"]) == 4
    # chance: predicting the majority class everywhere gives mIoU <= 1/4 (background IoU <= 1, the others 0)
    assert val[0]["mIoU"] > 0.6 and val[0]["aAcc"] > 0.8, val[0]


def test_cli_resume_continues_at_the_stored_iteration(voc, tmp_path, monkeypatch):
    work = tmp_path / "work"
    _run(_argv(voc, work, 30, ckpt=20, extra=("--no-validate",)), monkeypatch)
    assert torch.load(work / "iter_20.pth", map_location="cpu")["iter"] == 20
    _run(_argv(voc, work, 40, ckpt=20, extra=("--no-validate", "--resume-from", str(work / "iter_20.pth"))), monkeypatch)
    logs = sorted(glob.glob(str(work / "*.log.json")))
    starts = [json.loads(open(p).readline())["start_iter"] for p in logs]
    assert 20 in starts
    assert torch.load(work / "latest.pth", map_location="cpu")["iter"] == 40
    assert os.path.isfile(work / "iter_40.pth")


def test_cli_with_denoiser_and_distilled_backbones(voc, tmp_path, monkeypatch):
    import dvt.models as DVT
    torch.manual_seed(1)
    den = DVT.Denoiser(37, 37, 384, vit=None, num_blocks=1)
    torch.save({"denoiser": den.state_dict(), "optimizer": {}, "step": 0}, tmp_path / "denoiser.pth")
    vit = DVT.PretrainedViTWrapper(IDENT, stride=14, allow_random_init=True)
    torch.save({"model": vit.state_dict(), "optimizer": {}, "step": 0}, tmp_path / "distilled.pth")
    for flag, path in (("--load-denoiser-from", "denoiser.pth"), ("--load-distilled-model-from", "distilled.pth")):
        work = tmp_path / flag.strip("-")
        _run(_argv(voc, work, 40, extra=(flag, str(tmp_path / path))), monkeypatch)
        _, val = _val_records(work)
        assert len(val) == 1 and np.isfinite(val[0]["mIoU"]) and val[0]["aAcc"] > 0.3, val
        assert os.path.isfile(work / "iter_40.pth")


def test_cli_deterministic_runs_are_bit_identical(voc, tmp_path, monkeypatch):
    heads, metrics = [], []
    for run in range(2):
        work = tmp_path / f"det{run}"
        _run(_argv(voc, work, 30, extra=("--deterministic",)), monkeypatch)
        heads.append(torch.load(work / "latest.pth", map_location="cpu")["state_dict"])
        recs, val = _val_records(work)
        metrics.append([r for r in recs if r.get("mode") in ("train", "val")])
    assert heads[0].keys() == heads[1].keys()
    for k in heads[0]:
        assert torch.equal(heads[0][k], heads[1][k]), k
    assert metrics[0] == metrics[1]


def test_evaluation_in_workers_equals_serial(voc):
    """Validation images are decoded in DataLoader workers; the metrics do not depend on the worker count."""
    import dvt.models as DVT
    from dvt.dense_eval import config as C
    from dvt.dense_eval.data import SegDataset
    from dvt.dense_eval.model import LinearSegHead, ProbeBackbone
    from dvt.dense_eval.trainer import evaluate
    cfg = C.load_config(str(voc / "voc_linear.py"))
    C.merge_options(cfg, {"data.val.data_root": str(voc)})
    torch.manual_seed(0)
    vit = DVT.PretrainedViTWrapper(IDENT, stride=14, allow_random_init=True).cuda().eval()
    backbone = ProbeBackbone(vit, [8, 9, 10, 11], [3])
    head = LinearSegHead(384, 4).cuda()
    ds = SegDataset(cfg["data"]["val"], 4, train=False)
    test_cfg = cfg["model"]["test_cfg"]
    serial = evaluate(backbone, head, ds, test_cfg, 4, torch.device("cuda"), workers=0)
    pooled = evaluate(backbone, head, ds, test_cfg, 4, torch.device("cuda"), workers=2)
    assert serial == pooled and 0.0 <= serial["aAcc"] <= 1.0
