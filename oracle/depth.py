"""Float64 CPU restatement of the NYU depth probe in the reference's order (evaluation/depth: BNHead.depth_pred,
DepthBaseDecodeHead.losses, SigLoss, GradientLoss, DepthEncoderDecoder.encode_decode / aug_test, NYUDataset.eval_mask,
core/evaluation/metrics.py calculate), used as the yardstick of the dvt_depth_* kernels."""
import numpy as np
import torch
import torch.nn.functional as F

EPS = 1e-3


def head_forward(feat, cls, weight, bias, bins, up):
    """feat [B, C, h, w], cls [B, C] -> depth [B, 1, h up, w up]: upsample cat(feat, cls expanded) (bilinear,
    align_corners=False), 1x1 conv, relu + 0.1, normalise over the bins, expectation over bins."""
    x = torch.cat([feat, cls[:, :, None, None].expand_as(feat)], 1)
    x = F.interpolate(x, size=[s * up for s in feat.shape[2:]], mode="bilinear", align_corners=False)
    logit = torch.einsum("bchw,kc->bkhw", x, weight.reshape(weight.shape[0], -1)) + bias[None, :, None, None]
    logit = torch.relu(logit) + 0.1
    logit = logit / logit.sum(dim=1, keepdim=True)
    return torch.einsum("ikmn,k->imn", logit, bins).unsqueeze(1)


def sig_loss(pred, gt, warm_up):
    """SigLoss(valid_mask=True), eps 1e-3, boolean indexing as the reference."""
    m = gt > 0
    g = torch.log(pred[m] + EPS) - torch.log(gt[m] + EPS)
    if warm_up:
        return torch.sqrt(0.15 * torch.pow(torch.mean(g), 2))
    return torch.sqrt(torch.var(g) + 0.15 * torch.pow(torch.mean(g), 2))


def gradient_loss(pred, gt):
    """GradientLoss(valid_mask=True) on [B, 1, H, W] as the reference indexes it (batch and channel dimensions)."""
    total = 0
    for i in range(4):
        inp = pred if i == 0 else pred[::2 * i, ::2 * i]
        tgt = gt if i == 0 else gt[::2 * i, ::2 * i]
        mask = tgt > 0
        n = torch.sum(mask)
        ldd = torch.mul(torch.log(inp + EPS) - torch.log(tgt + EPS), mask)
        v = torch.mul(torch.abs(ldd[0:-2, :] - ldd[2:, :]), torch.mul(mask[0:-2, :], mask[2:, :]))
        h = torch.mul(torch.abs(ldd[:, 0:-2] - ldd[:, 2:]), torch.mul(mask[:, 0:-2], mask[:, 2:]))
        total = total + (torch.sum(h) + torch.sum(v)) / n
    return total


def loss(depth4, gt, warm_up, grad_weight=0.5):
    """decode.loss_depth + decode.loss_grad of the head's depth [B, 1, h up, w up] against gt [B, 1, H, W]."""
    pred = F.interpolate(depth4, size=gt.shape[2:], mode="bilinear", align_corners=False)
    ld = sig_loss(pred, gt, warm_up)
    lg = grad_weight * gradient_loss(pred, gt)
    return ld, lg, ld + lg


def aug_predict(maps, flips, size, min_depth, max_depth):
    """maps [n_aug, 1, Hu, Wu] -> the aug_test prediction [Ho, Wo]: clamp, resize, un-flip, sum, / n_aug."""
    out = 0
    for m, f in zip(maps, flips):
        p = F.interpolate(torch.clamp(m[None], min_depth, max_depth), size=size, mode="bilinear", align_corners=False)
        out = out + (p.flip(dims=(3,)) if f else p)
    return (out / len(maps))[0, 0]


def eval_mask(gt, min_depth, max_depth, crop):
    m = (gt > min_depth) & (gt < max_depth)
    box = np.zeros_like(m)
    y0, y1, x0, x1 = crop
    box[y0:y1, x0:x1] = True
    return m & box


def calculate(gt, pred):
    """core/evaluation/metrics.py calculate(): (a1, a2, a3, abs_rel, rmse, log_10, rmse_log, silog, sq_rel)."""
    if gt.shape[0] == 0:
        return np.full(9, np.nan)
    thresh = np.maximum(gt / pred, pred / gt)
    a1, a2, a3 = (thresh < 1.25).mean(), (thresh < 1.25 ** 2).mean(), (thresh < 1.25 ** 3).mean()
    abs_rel = np.mean(np.abs(gt - pred) / gt)
    sq_rel = np.mean(((gt - pred) ** 2) / gt)
    rmse = np.sqrt(((gt - pred) ** 2).mean())
    rmse_log = np.sqrt(((np.log(gt) - np.log(pred)) ** 2).mean())
    err = np.log(pred) - np.log(gt)
    with np.errstate(invalid="ignore"):
        silog = np.sqrt(np.mean(err ** 2) - np.mean(err) ** 2) * 100
    if np.isnan(silog):
        silog = 0
    log_10 = np.abs(np.log10(gt) - np.log10(pred)).mean()
    return np.array([a1, a2, a3, abs_rel, rmse, log_10, rmse_log, silog, sq_rel], dtype=np.float64)


def image_metrics(maps, flips, gt, min_depth, max_depth, crop):
    """One image's nine metrics: aug_test prediction, eval mask, calculate (float64 throughout)."""
    pred = aug_predict(torch.as_tensor(maps, dtype=torch.float64), flips, gt.shape, min_depth, max_depth).numpy()
    gt = np.asarray(gt, dtype=np.float64)
    m = eval_mask(gt, min_depth, max_depth, crop)
    return calculate(gt[m], pred[m])
