"""The four-layer linear probes (in_index [0, 1, 2, 3] of out_indices [8, 9, 10, 11], DINOv2's standard linear protocol)
on the GPU: the segmentation head's loss and gradients against a float64 oracle of BatchNorm + 1x1 conv over the
concatenated layers, the depth head's losses with one cls token per layer against the oracle/depth.py restatement, and
evaluate_dense_tasks.py / evaluate_depth.py end to end with the four-layer head, twice under --deterministic."""
import glob
import json

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_dense_eval_gpu as SEG
import test_depth_probe_gpu as DEP
from oracle import depth as OD

pytestmark = pytest.mark.gpu

IDENT = "vit_small_patch14_dinov2.lvd142m"
C = 384
LAYERS = [8, 9, 10, 11]


@pytest.fixture(scope="module")
def voc(tmp_path_factory):
    return SEG.voc.__wrapped__(tmp_path_factory)


@pytest.fixture(scope="module")
def nyu(tmp_path_factory):
    return DEP.nyu.__wrapped__(tmp_path_factory)


@pytest.fixture(scope="module")
def vit():
    import dvt.models as DVT
    from oracle import vit as OV
    cfg = OV.CONFIGS[IDENT]
    w = DVT.PretrainedViTWrapper(IDENT, stride=14, allow_random_init=True)
    w.model.load_state_dict(OV.random_state_dict(cfg, seed=0))     # LayerScale U(0.5, 1.5): the layers differ
    return w.cuda().eval()


def _voc_batch(voc, n=4, H=210, W=252):
    """n images of the VOC fixture, cropped to H x W (whole patches) and normalised, with their labels."""
    from PIL import Image
    names = (voc / "ImageSets/Segmentation/train.txt").read_text().split()[:n]
    mean, std = torch.tensor([123.675, 116.28, 103.53]), torch.tensor([58.395, 57.12, 57.375])
    imgs, segs = [], []
    for name in names:
        img = torch.from_numpy(np.asarray(Image.open(voc / "JPEGImages" / f"{name}.jpg"), dtype=np.float32))[:H, :W]
        imgs.append(((img - mean) / std).permute(2, 0, 1))
        segs.append(torch.from_numpy(np.asarray(Image.open(voc / "SegmentationClass" / f"{name}.png")))[:H, :W])
    return torch.stack(imgs).cuda(), torch.stack(segs).cuda()


def _per_layer(vit, x, norm, prefix):
    """The maps (and cls rows) of LAYERS from one get_intermediate_layers call per layer."""
    outs = [vit.get_intermediate_layers(x, n=[l], reshape=True, return_prefix_tokens=prefix, norm=norm)[0] for l in LAYERS]
    if not prefix:
        return [o.permute(0, 2, 3, 1) for o in outs], None
    return [o[0].permute(0, 2, 3, 1) for o in outs], [o[1][:, 0] for o in outs]


def test_four_layer_segmentation_head_matches_float64(voc, vit):
    from dvt.dense_eval import seg_ops
    from dvt.dense_eval.model import LinearSegHead, ProbeBackbone
    x, seg = _voc_batch(voc)
    probe = ProbeBackbone(vit, LAYERS, [0, 1, 2, 3])
    feats = probe(x)
    maps, _ = _per_layer(vit, x, False, False)
    assert feats.shape == (4, 15, 18, 4 * C) and torch.equal(feats, torch.cat(maps, -1))
    K = 4
    torch.manual_seed(0)
    head = LinearSegHead(4 * C, K).cuda().train()
    with torch.no_grad():
        head.bn.weight.copy_(torch.rand(4 * C) + 0.5)
        head.bn.bias.copy_(torch.randn(4 * C) * 0.1)
        head.conv_seg.weight.normal_(0, 0.05)
    logits = head(feats)
    logits.retain_grad()
    loss = seg_ops.upsample_cross_entropy(logits, seg)
    loss.backward()
    # float64: BatchNorm2d in training mode (batch statistics, biased variance), 1x1 conv, mmseg's loss
    f64 = torch.cat([m.double() for m in maps], -1).permute(0, 3, 1, 2)
    g64 = head.bn.weight.detach().double().requires_grad_(True)
    b64 = head.bn.bias.detach().double().requires_grad_(True)
    w64 = head.conv_seg.weight.detach().double().requires_grad_(True)
    cb64 = head.conv_seg.bias.detach().double().requires_grad_(True)
    mu, var = f64.mean((0, 2, 3), keepdim=True), f64.var((0, 2, 3), unbiased=False, keepdim=True)
    y = (f64 - mu) / torch.sqrt(var + head.bn.eps) * g64[:, None, None] + b64[:, None, None]
    lo64 = F.conv2d(y, w64, cb64)
    lo64.retain_grad()
    up = F.interpolate(lo64, size=seg.shape[-2:], mode="bilinear", align_corners=False)
    ref = F.cross_entropy(up, seg.long(), reduction="none", ignore_index=255).mean()
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 1e-4 * abs(ref.item())
    assert torch.isfinite(lo64.grad).all() and lo64.grad.abs().max() > 0

    def rel(a, b):
        return ((a.double() - b).norm() / b.norm()).item()

    assert rel(logits.grad.permute(0, 3, 1, 2), lo64.grad) < 1e-4
    for got, want in ((head.conv_seg.weight.grad, w64.grad), (head.conv_seg.bias.grad, cb64.grad),
                      (head.bn.weight.grad, g64.grad), (head.bn.bias.grad, b64.grad)):
        assert rel(got, want) < 1e-4


def test_four_layer_depth_head_with_cls_per_layer_matches_oracle(voc, vit):
    from dvt.dense_eval import depth_ops as O
    from dvt.dense_eval.depth import DepthHead, depth_losses
    from dvt.dense_eval.model import ProbeBackbone
    x, _ = _voc_batch(voc, n=3)
    probe = ProbeBackbone(vit, LAYERS, [0, 1, 2, 3], return_cls=True, norm=True)
    feats, cls = probe(x)
    maps, clss = _per_layer(vit, x, True, True)
    assert torch.equal(feats, torch.cat(maps, -1)) and torch.equal(cls, torch.cat(clss, -1)) and cls.shape == (3, 4 * C)
    K, up = 256, 4
    torch.manual_seed(0)
    head = DepthHead(8 * C, K, 0.001, 10, up, n_maps=4).cuda()
    B, h, w = feats.shape[:3]
    g = torch.Generator().manual_seed(0)
    gt = torch.rand(B, 14 * h - 4, 14 * w - 2, generator=g) * 9 + 0.5
    gt[torch.rand(gt.shape, generator=g) < 0.1] = 0
    losses = depth_losses(head(feats, cls), gt.cuda(), O.SigLossState(warm_up=False), 1.0, 0.5)
    # the reference's BNHead: per layer cat(map, cls expanded), the layers concatenated (resize_concat), then depth_pred
    xs = torch.cat([torch.cat([m.cpu().double().permute(0, 3, 1, 2), c.cpu().double()[:, :, None, None].expand(B, C, h, w)],
                              1) for m, c in zip(maps, clss)], 1)
    xs = F.interpolate(xs, size=[h * up, w * up], mode="bilinear", align_corners=False)
    wt = head.conv_depth.weight.detach().cpu().double().reshape(K, -1)
    bias = head.conv_depth.bias.detach().cpu().double()
    logit = torch.relu(torch.einsum("bchw,kc->bkhw", xs, wt) + bias[None, :, None, None])
    logit = (logit + 0.1) / (logit + 0.1).sum(dim=1, keepdim=True)
    d4 = torch.einsum("ikmn,k->imn", logit, torch.linspace(0.001, 10, K, dtype=torch.float64)).unsqueeze(1)
    ld, lg, tot = OD.loss(d4, gt.double()[:, None], warm_up=False)
    assert losses["loss"].item() == pytest.approx(tot.item(), rel=1e-4)
    assert losses["decode.loss_depth"].item() == pytest.approx(ld.item(), rel=1e-4)
    assert losses["decode.loss_grad"].item() == pytest.approx(lg.item(), rel=1e-4, abs=1e-7)


FOUR = ["model.decode_head.in_index=[0,1,2,3]", f"model.decode_head.in_channels=[{C},{C},{C},{C}]"]


def _seg_argv(voc, work, extra=()):
    return SEG._argv(voc, work, 20, extra=(*FOUR, f"model.decode_head.channels={4 * C}", *extra))


def _depth_argv(nyu, work, extra=()):
    return DEP._argv(nyu, work, 10, ckpt=10, evaluate=10,
                     extra=(*FOUR, f"model.decode_head.channels={8 * C}", "model.backbone.out_indices=[8,9,10,11]", *extra))


def test_segmentation_cli_with_the_four_layer_head(voc, tmp_path, monkeypatch):
    work = tmp_path / "work"
    SEG._run(_seg_argv(voc, work), monkeypatch)
    ck = torch.load(work / "latest.pth", map_location="cpu")
    sd = ck["state_dict"]
    assert ck["iter"] == 20
    for k in ("weight", "bias", "running_mean", "running_var"):
        assert sd[f"decode_head.bn.{k}"].shape == (4 * C,)
    assert sd["decode_head.conv_seg.weight"].shape == (4, 4 * C, 1, 1)
    recs, val = SEG._val_records(work)
    assert all(np.isfinite(r["loss"]) for r in recs if r.get("mode") == "train")
    assert len(val) == 1 and val[0]["iter"] == 20 and np.isfinite(val[0]["mIoU"]) and len(val[0]["IoU"]) == 4


def test_depth_cli_with_the_four_layer_head(nyu, tmp_path, monkeypatch):
    work = tmp_path / "work"
    DEP._run(_depth_argv(nyu, work), monkeypatch)
    ck = torch.load(work / "latest.pth", map_location="cpu")
    assert ck["state_dict"]["decode_head.conv_depth.weight"].shape == (256, 8 * C, 1, 1)   # 4 x (patch tokens + cls)
    recs = DEP._records(work)
    val = [r for r in recs if r.get("mode") == "val"]
    assert len(val) == 1 and all(np.isfinite(val[0][k]) for k in ("a1", "abs_rel", "rmse", "silog"))
    assert all(np.isfinite(r["loss"]) for r in recs if r.get("mode") == "train")


@pytest.mark.parametrize("task", ["seg", "depth"])
def test_deterministic_four_layer_runs_are_bit_identical(task, voc, nyu, tmp_path, monkeypatch):
    heads, logs = [], []
    for run in range(2):
        work = tmp_path / f"det{run}"
        if task == "seg":
            SEG._run(_seg_argv(voc, work, extra=("--deterministic",)), monkeypatch)
        else:
            DEP._run(_depth_argv(nyu, work, extra=("--deterministic",)), monkeypatch)
        heads.append(torch.load(work / "latest.pth", map_location="cpu")["state_dict"])
        (log,) = glob.glob(str(work / "*.log.json"))
        logs.append([r for r in map(json.loads, open(log)) if r.get("mode") in ("train", "val")])
    assert heads[0].keys() == heads[1].keys() and all(torch.equal(heads[0][k], heads[1][k]) for k in heads[0])
    assert logs[0] and logs[0] == logs[1]
