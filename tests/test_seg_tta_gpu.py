"""Segmentation probe, test-time augmentation on the GPU: the per-augmentation kernel (resize of preds / count, softmax,
un-flip, sum) against float64 torch, the argmax / histogram kernel, multi-scale + flip inference of one image against a
torch restatement of mmseg's slide_inference + aug_test, repeatability, evaluation through the single-scale and the
augmented paths, and evaluate_dense_tasks.py end to end with ms+flip enabled through --cfg-options."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_dense_eval_gpu import IDENT, _argv, _hist_np, _labels, _run, _val_records, voc  # noqa: F401

pytestmark = pytest.mark.gpu

RATIOS = [0.5, 0.75, 1.0, 1.25, 1.5, 1.75]


def _acc_count(K, Hc, Wc, seed):
    """Slide-inference sums: a smooth field of logits (window logits are upsampled from the patch grid) times the window
    count.  On rough fields the fp32 source coordinates of ATen's resize, which the kernel reproduces, move the result
    by more than 1e-5 from the float64 resize at these sizes."""
    g = torch.Generator().manual_seed(seed)
    count = torch.randint(1, 5, (Hc, Wc), generator=g).float()
    field = torch.randn(1, K, Hc // 6 + 2, Wc // 6 + 2, generator=g) * 3
    acc = F.interpolate(field, size=(Hc, Wc), mode="bilinear", align_corners=False)[0] * count
    return acc.cuda(), count.cuda()


def _aug_ref(acc, count, flip, out_size):
    """mmseg: resize(preds / count_mat, ori_shape), softmax over the classes, flip back; in float64."""
    mean = acc.double() / count.double()
    p = F.softmax(F.interpolate(mean[None], size=out_size, mode="bilinear", align_corners=False)[0], dim=0)
    return p.flip(2) if flip else p


@pytest.mark.parametrize("K", [21, 150])
@pytest.mark.parametrize("Hc, Wc, Ho, Wo", [
    (41, 57, 75, 101),        # augmentation smaller than the original
    (75, 101, 75, 101),       # equal
    (131, 177, 75, 101),      # larger
    (33, 250, 97, 63),        # odd sizes, smaller in one axis and larger in the other
    (1, 1, 5, 7),
])
@pytest.mark.parametrize("flip", [False, True])
def test_aug_accumulate_matches_float64(K, Hc, Wc, Ho, Wo, flip):
    from dvt.dense_eval import seg_ops
    acc, count = _acc_count(K, Hc, Wc, seed=K + Hc * 7 + Wo)
    prob0 = torch.rand(K, Ho, Wo, generator=torch.Generator().manual_seed(1)).cuda()
    ref = prob0.double() + _aug_ref(acc, count, flip, (Ho, Wo))
    acc_in, count_in = acc.clone(), count.clone()
    outs = []
    for _ in range(3):
        prob = prob0.clone()
        seg_ops.aug_accumulate(acc, count, flip, prob)
        outs.append(prob)
    err = (outs[0].double() - ref).norm() / ref.norm()
    assert err <= 1e-5, err.item()
    assert (outs[0].double() - ref).abs().max() <= 1e-5 * ref.abs().max()
    assert torch.equal(outs[1], outs[0]) and torch.equal(outs[2], outs[0])
    assert torch.equal(acc, acc_in) and torch.equal(count, count_in)


@pytest.mark.parametrize("K", [2, 40, 80, 255])           # the other register-array widths (KV = 1, 2, 3, 8)
def test_aug_accumulate_class_counts(K):
    from dvt.dense_eval import seg_ops
    acc, count = _acc_count(K, 29, 38, seed=K)
    prob = torch.zeros(K, 45, 31, device="cuda")
    seg_ops.aug_accumulate(acc, count, True, prob)
    seg_ops.aug_accumulate(acc, count, False, prob)
    ref = _aug_ref(acc, count, True, (45, 31)) + _aug_ref(acc, count, False, (45, 31))
    assert (prob.double() - ref).abs().max() <= 1e-5 * ref.abs().max()
    assert torch.allclose(prob.sum(0).double(), torch.full_like(ref[0], 2.0), atol=1e-5)


def test_aug_argmax_hist_divides_then_takes_the_lowest_tied_class():
    from dvt.dense_eval import seg_ops
    K, Ho, Wo, n = 7, 33, 45, 3
    g = torch.Generator().manual_seed(0)
    prob = torch.randint(0, 4, (K, Ho, Wo), generator=g).float().cuda()    # many exact ties
    gt = _labels(1, Ho, Wo, K, seed=3)[0]
    gt[0, :5] = K + 3                                                       # >= K: counted as a prediction only
    hist = torch.zeros(4, K, dtype=torch.int64, device="cuda")
    seg_ops.aug_argmax_hist(prob, n, gt, hist)
    pred = (prob / n).argmax(0)
    assert np.array_equal(hist.cpu().numpy(), _hist_np(pred.cpu().numpy(), gt.cpu().numpy(), K))


# ---------------------------------------------------------------------------------------------------------------------
# one image, multi-scale + flip
# ---------------------------------------------------------------------------------------------------------------------
def _logits_fn(K, seed):
    from dvt.models import CenterPadding
    g = torch.Generator().manual_seed(seed)
    w1 = (torch.randn(32, 3, 14, 14, generator=g) * 0.1).cuda()
    w2 = torch.randn(K, 32, generator=g).cuda()
    pad = CenterPadding(14)

    def fn(crops):                              # a random "backbone + head": NHWC logits at patch resolution
        f = torch.tanh(F.conv2d(pad(crops), w1, stride=14)).permute(0, 2, 3, 1)
        return f @ w2.t()
    return fn


def _augs(Ho, Wo, seed):
    """ms+flip augmentations of a smooth random image: keep-ratio resizes of (Ho, Wo) into (int(1024 r), int(Ho r))."""
    from dvt.dense_eval.data import rescale_size
    g = torch.Generator().manual_seed(seed)
    img = F.interpolate(torch.randn(1, 3, Ho // 8 + 1, Wo // 8 + 1, generator=g), size=(Ho, Wo), mode="bilinear",
                        align_corners=False).cuda()
    augs = []
    for r in RATIOS:
        a = F.interpolate(img, size=rescale_size(Ho, Wo, (int(1024 * r), int(Ho * r))), mode="bilinear",
                          align_corners=False)[0]
        augs += [(a.contiguous(), False), (a.flip(2).contiguous(), True)]
    return augs


def _mmseg_aug_test_torch(logits_fn, augs, crop, stride, K, out_size):
    """mmseg 0.27 slide_inference (one window at a time) + inference (resize, softmax, flip) + aug_test (sum, / n), with
    the logits in float32 as the model gives them and everything after them in float64."""
    from dvt.dense_eval.data import slide_windows
    total = 0
    for img, flip in augs:
        H, W = img.shape[1:]
        preds = torch.zeros(1, K, H, W, device=img.device, dtype=torch.float64)
        count = torch.zeros(1, 1, H, W, device=img.device, dtype=torch.float64)
        for (y1, y2, x1, x2) in slide_windows(H, W, crop, stride):
            cl = logits_fn(img[None, :, y1:y2, x1:x2]).permute(0, 3, 1, 2).double()
            cl = F.interpolate(cl, size=(y2 - y1, x2 - x1), mode="bilinear", align_corners=False)
            preds += F.pad(cl, (x1, W - x2, y1, H - y2))
            count[:, :, y1:y2, x1:x2] += 1
        out = F.softmax(F.interpolate(preds / count, size=out_size, mode="bilinear", align_corners=False), dim=1)
        total = total + (out.flip(3) if flip else out)
    return (total / len(augs))[0]


@pytest.mark.parametrize("K", [21, 150])
def test_ms_flip_inference_matches_mmseg_aug_test(K):
    from dvt.dense_eval import seg_ops
    Ho, Wo = 181, 243
    fn, augs = _logits_fn(K, seed=K), _augs(Ho, Wo, seed=K + 1)
    # smaller than the crop (one window) up to 20 windows
    assert [tuple(a.shape[1:]) for a, _ in augs[::2]] == [(90, 121), (135, 181), (181, 243), (226, 303), (271, 364),
                                                          (316, 424)]
    gt = _labels(1, Ho, Wo, K, seed=5)[0]
    crop, stride = (128, 128), (85, 85)
    ref = _mmseg_aug_test_torch(fn, augs, crop, stride, K, (Ho, Wo))
    top2 = ref.topk(2, dim=0).values
    n_ties = int((((top2[0] - top2[1]) < 1e-5) & (gt != 255)).sum())
    ref_hist = _hist_np(ref.argmax(0).cpu().numpy(), gt.cpu().numpy(), K)
    hists = []
    for _ in range(3):
        hist = torch.zeros(4, K, dtype=torch.int64, device="cuda")
        seg_ops.aug_slide_inference_hist(fn, augs, gt, K, crop, stride, hist, max_batch=4)
        hists.append(hist)
    assert torch.equal(hists[1], hists[0]) and torch.equal(hists[2], hists[0])
    diff = np.abs(hists[0].cpu().numpy() - ref_hist)
    assert diff.sum() <= 6 * n_ties, (diff.sum(), n_ties)     # one pixel moves at most 1 + 2 + 2 + 0 histogram counts
    assert hists[0][2].sum().item() == int((gt != 255).sum())
    assert hists[0][3].sum().item() == int(((gt != 255) & (gt < K)).sum())
    # batching windows across augmentations does not change the result
    hist1 = torch.zeros(4, K, dtype=torch.int64, device="cuda")
    seg_ops.aug_slide_inference_hist(fn, augs, gt, K, crop, stride, hist1, max_batch=1)
    assert np.abs(hist1.cpu().numpy() - hists[0].cpu().numpy()).sum() <= 6 * n_ties


# ---------------------------------------------------------------------------------------------------------------------
# evaluation: the single-scale and the augmented paths, and the command line
# ---------------------------------------------------------------------------------------------------------------------
def _probe(voc, options):
    import dvt.models as DVT
    from dvt.dense_eval import config as C
    from dvt.dense_eval.data import SegDataset
    from dvt.dense_eval.model import LinearSegHead, ProbeBackbone
    cfg = C.load_config(str(voc / "voc_linear.py"))
    C.merge_options(cfg, dict({"data.val.data_root": str(voc)}, **options))
    torch.manual_seed(0)
    vit = DVT.PretrainedViTWrapper(IDENT, stride=14, allow_random_init=True).cuda().eval()
    backbone = ProbeBackbone(vit, [8, 9, 10, 11], [3])
    head = LinearSegHead(384, 4).cuda().eval()
    fn = lambda crops: head(backbone(crops))  # noqa: E731
    return backbone, head, fn, SegDataset(cfg["data"]["val"], 4, train=False), cfg["model"]["test_cfg"]


@pytest.mark.parametrize("ms_flip", [False, True])
@torch.no_grad()
def test_evaluate_dispatches_on_the_number_of_augmentations(voc, ms_flip):
    from dvt.dense_eval import seg_ops
    from dvt.dense_eval.metrics import metrics_from_hist
    from dvt.dense_eval.trainer import evaluate
    opts = {"data.val.pipeline.1.img_ratios": RATIOS, "data.val.pipeline.1.flip": True} if ms_flip else {}
    backbone, head, fn, ds, test_cfg = _probe(voc, opts)
    assert len(ds.augs) == (12 if ms_flip else 1)
    hist = torch.zeros(4, 4, dtype=torch.int64, device="cuda")
    for i in range(len(ds)):
        img, gt = ds[i]
        if ms_flip:
            augs = [(a.cuda(), f) for a, f in img]
            seg_ops.aug_slide_inference_hist(fn, augs, gt.cuda(), 4, test_cfg["crop_size"], test_cfg["stride"], hist)
        else:
            seg_ops.slide_inference_hist(fn, img.cuda(), gt.cuda(), 4, test_cfg["crop_size"], test_cfg["stride"], hist)
    # evaluate's DataLoader (pinned items) gives the histograms of the loop above.  Both decode in this process: torch's
    # CPU bilinear resize of the test pipeline can round a few uint8 pixels differently under another thread count.
    assert evaluate(backbone, head, ds, test_cfg, 4, torch.device("cuda"), workers=0) == metrics_from_hist(hist.cpu().numpy())


def test_cli_ms_flip_evaluation_is_finite_and_deterministic(voc, tmp_path, monkeypatch):
    extra = ("--deterministic", "--cfg-options", "data.val.pipeline.1.img_ratios=[0.5,0.75,1.0,1.25,1.5,1.75]",
             "data.val.pipeline.1.flip=True")
    vals = []
    for run in range(2):
        work = tmp_path / f"ms{run}"
        _run(_argv(voc, work, 20, extra=extra), monkeypatch)
        _, val = _val_records(work)
        assert len(val) == 1 and os.path.isfile(work / "iter_20.pth")
        assert all(math.isfinite(val[0][k]) and 0.0 <= val[0][k] <= 1.0 for k in ("mIoU", "mAcc", "aAcc")), val[0]
        vals.append(val[0])
    assert vals[0] == vals[1]
