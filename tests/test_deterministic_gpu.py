"""Deterministic training (torch.use_deterministic_algorithms) on the GPU: every fixed-order kernel that replaces a
float-atomic reduction of the stage-2 / stage-3 backward -- the query-major dQ kernel of the attention backward, ordered
split-K weight gradients, column sums, the LayerNorm backward, the loss and the position-embedding resample backward --
against the atomic path and an fp32 / float64 reference, bit-identical repeats, and end-to-end runs (parameters, both
AdamW moments and logged losses `torch.equal` over two runs, with and without gradient checkpointing), the gradients
against the fp32 oracle and both trainers' `--deterministic` flag."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def det():
    """Deterministic mode for the test; the previous setting is always restored."""
    prev, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=warn)


def _cos(a, b):
    return F.cosine_similarity(a.flatten().double(), b.flatten().double(), dim=0).item()


def _dev_ok():
    from dvt import _lib
    torch.cuda.synchronize()
    assert _lib.device_error() == 0


def _atomic(fn, *a):
    """fn(*a) with deterministic mode off (the existing atomic kernels)."""
    torch.use_deterministic_algorithms(False)
    try:
        return fn(*a)
    finally:
        torch.use_deterministic_algorithms(True)


# ---------------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hd", [64, 80])
@pytest.mark.parametrize("B,N,heads", [(2, 257, 2), (1, 1029, 3), (1, 1370, 2), (3, 100, 1)])
def test_attention_dq_kernel(det, hd, B, N, heads):
    from dvt import train_ops
    g = torch.Generator(device="cuda").manual_seed(N + heads + hd)
    C = heads * hd
    qkv = (torch.randn(B, N, 3 * C, device="cuda", generator=g) * 1.2).bfloat16()
    dout = torch.randn(B, N, C, device="cuda", generator=g).bfloat16()
    out, lse = train_ops.attention_fwd_lse(qkv, heads, hd)
    runs = [train_ops.attention_bwd(qkv, out, dout, lse, heads, hd) for _ in range(3)]
    ref_atomic = _atomic(train_ops.attention_bwd, qkv, out, dout, lse, heads, hd)
    _dev_ok()
    assert all(torch.equal(runs[0], r) for r in runs[1:])                          # bit-identical repeats
    assert torch.equal(runs[0][..., C:], ref_atomic[..., C:])                        # dK, dV: the same kernel's bits
    # fp32 autograd reference on the CPU (cuBLAS would refuse under the flag)
    x = qkv.float().cpu().requires_grad_(True)
    q, k, v = x.reshape(B, N, 3, heads, hd).permute(2, 0, 3, 1, 4).unbind(0)
    s = (q @ k.transpose(-1, -2)) * hd ** -0.5
    (s.softmax(-1) @ v).transpose(1, 2).reshape(B, N, C).backward(dout.float().cpu())
    dq, dq_atomic, dq_ref = runs[0][..., :C].float().cpu(), ref_atomic[..., :C].float().cpu(), x.grad[..., :C]
    assert _cos(dq, dq_ref) > 0.998 and (dq - dq_ref).abs().max().item() < 0.03 * dq_ref.abs().max().item() + 1e-3
    assert _cos(dq, dq_atomic) > 0.999 and (dq - dq_atomic).abs().max().item() < 0.02 * dq_atomic.abs().max().item() + 1e-3


@pytest.mark.parametrize("rows,n_out,n_in", [(8192, 768, 768), (5000, 384, 1536), (2738, 2304, 768)])
def test_ordered_split_k(det, rows, n_out, n_in):
    from dvt import train_ops
    from dvt._lib import check, cur_stream, lib, ptr
    g = torch.Generator(device="cuda").manual_seed(rows)
    dy = torch.randn(rows, n_out, device="cuda", generator=g).bfloat16()
    x = torch.randn(rows, n_in, device="cuda", generator=g).bfloat16()
    splits = train_ops.wgrad_splits(rows, n_out, n_in)
    assert splits > 1
    a, b = train_ops.wgrad(dy, x), train_ops.wgrad(dy, x)
    # the K-slice partials as separate splits = 1 GEMMs (same k-block ranges as the split-K launch), added in order
    kb = (rows + 63) // 64
    per = (kb + splits - 1) // splits
    acc = None
    for s in range(splits):
        r0, r1 = min(rows, s * per * 64), min(rows, (s + 1) * per * 64)
        part = torch.zeros(n_out, n_in, device="cuda")
        if r1 > r0:
            check(lib().dvt_gemm_bf16_wgrad_ordered(ptr(dy[r0:r1]), n_out, ptr(x[r0:r1]), n_in, n_out, n_in, r1 - r0, ptr(part),
                                                    n_in, 1, None, cur_stream()), "wgrad slice")
        acc = part if acc is None else acc + part
    atomic = _atomic(train_ops.wgrad, dy, x)
    _dev_ok()
    assert torch.equal(a, b) and torch.equal(a, acc)
    assert (a - atomic).abs().max().item() < 1e-4 * atomic.abs().max().item()


def test_colsum_layernorm_loss(det):
    from dvt import train_ops
    g = torch.Generator(device="cuda").manual_seed(5)
    rows, C = 4100, 768
    for t in (torch.randn(rows, 3 * C, device="cuda", generator=g).bfloat16(), torch.randn(rows, C, device="cuda", generator=g)):
        a, b = train_ops.colsum(t), train_ops.colsum(t)
        ref = _atomic(train_ops.colsum, t)
        assert torch.equal(a, b) and (a - ref).abs().max().item() < 1e-5 * t.float().abs().sum(0).max().item()
    x = torch.randn(rows, C, device="cuda", generator=g) * 2 + 0.5
    w = 1 + 0.2 * torch.randn(C, device="cuda", generator=g)
    dy = torch.randn(rows, C, device="cuda", generator=g)
    acc0 = torch.randn(rows, C, device="cuda", generator=g)
    outs = []
    for _ in range(2):
        acc = acc0.clone()
        outs.append((acc,) + train_ops.layernorm_bwd_(acc, x, w, dy))
    acc_r = acc0.clone()
    dg_r, db_r = _atomic(train_ops.layernorm_bwd_, acc_r, x, w, dy)
    assert all(torch.equal(p, q) for p, q in zip(outs[0], outs[1]))
    assert torch.equal(outs[0][0], acc_r)                                  # dx: the same per-row arithmetic
    assert (outs[0][1] - dg_r).abs().max().item() < 1e-4 * dg_r.abs().max().item() + 1e-4
    assert (outs[0][2] - db_r).abs().max().item() < 1e-4 * db_r.abs().max().item() + 1e-4
    pred = torch.randn(8, 37, 37, C, device="cuda", generator=g)
    tgt = torch.randn(8, 37, 37, C, device="cuda", generator=g)
    l1, l2 = torch.stack(train_ops.denoise_loss(pred, tgt)), torch.stack(train_ops.denoise_loss(pred, tgt))
    lr = torch.stack(_atomic(train_ops.denoise_loss, pred, tgt))
    _dev_ok()
    assert torch.equal(l1, l2) and (l1 - lr).abs().max().item() < 1e-5


@pytest.mark.parametrize("src,dst", [((37, 37), (73, 73)), ((14, 14), (32, 32)), ((24, 24), (14, 14)), ((5, 7), (9, 4))])
def test_resample_backward(det, src, dst):
    from dvt import train_ops
    (gh, gw), (h, w) = src, dst
    C = 384
    gen = torch.Generator().manual_seed(gh * w)
    g64 = torch.randn(1, C, gh, gw, generator=gen, dtype=torch.float64)
    dout = torch.randn(1, C, h, w, generator=gen, dtype=torch.float64)
    grads, fwd = [], None
    for _ in range(2):
        gg = g64.float().cuda().requires_grad_(True)
        y = train_ops.resample_bicubic(gg, h, w)
        y.backward(dout.float().cuda())
        grads.append(gg.grad.clone())
        fwd = y.detach()
    _dev_ok()
    assert torch.equal(grads[0], grads[1])
    assert torch.equal(fwd, F.interpolate(g64.float().cuda(), size=(h, w), mode="bicubic", antialias=True))
    ref = g64.clone().requires_grad_(True)
    F.interpolate(ref, size=(h, w), mode="bicubic", antialias=True).backward(dout)         # float64 CPU autograd
    err = (grads[0].cpu().double() - ref.grad).abs().max().item()
    assert err < 1e-5 * ref.grad.abs().max().item() + 1e-5, err


# ---------------------------------------------------------------------------------------------------------------------
# end to end: two runs, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
def _state(opt, logs):
    return [opt.flat_p.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone(), torch.stack(logs)]


def _assert_same(a, b):
    for name, x, y in zip(("parameters", "exp_avg", "exp_avg_sq", "losses"), a, b):
        assert torch.equal(x, y), name


def test_stage2_denoiser_bit_identical(det):
    import dvt.models as DVT
    from dvt import train_ops
    from dvt.optim import FusedAdamW
    C, hw, B, T = 256, (9, 9), 4, 20
    torch.manual_seed(0)
    sd = {k: v.clone() for k, v in DVT.Denoiser(hw[0], hw[1], C, vit=None, num_blocks=1).state_dict().items()}
    g = torch.Generator().manual_seed(1)
    batches = [(torch.randn(B, 11, 13, C, generator=g), torch.randn(B, 11, 13, C, generator=g)) for _ in range(T)]  # resampled
    runs = []
    for _ in range(2):
        m = DVT.Denoiser(hw[0], hw[1], C, vit=None, num_blocks=1)
        m.load_state_dict(sd)
        m = m.cuda().train()
        opt = FusedAdamW(m.parameters(), lr=1e-3, weight_decay=1e-5)
        logs = []
        for x, t in batches:
            loss, l2, cs = train_ops.denoise_loss(m(x.cuda()), t.cuda())
            opt.zero_grad()
            loss.backward()
            opt.step()
            logs.append(torch.stack([loss.detach(), l2.detach(), cs.detach()]))
        runs.append(_state(opt, logs))
    _dev_ok()
    _assert_same(runs[0], runs[1])
    assert not torch.equal(runs[0][0], runs[0][0] * 0)


def _random_wrapper(ident, stride, depth):
    import re
    import dvt.models as DVT
    from dvt.models import vit_wrapper as VW
    a = dict(VW.ARCHS[ident])
    a["depth"] = depth
    P = int(re.search(r"patch(\d+)", ident).group(1))
    w = DVT.PretrainedViTWrapper(ident, stride=stride, allow_random_init=True)
    w.model = VW.B200VisionTransformer(ident, P, a)
    w.model.patch_embed.proj.stride = [stride, stride]
    gen = torch.Generator().manual_seed(7)
    with torch.no_grad():
        for name, p in w.model.named_parameters():
            if ".ls" in name:
                p.copy_(0.5 + torch.rand(p.shape, generator=gen))
            elif "norm" in name and name.endswith("weight"):
                p.copy_(1 + 0.1 * torch.randn(p.shape, generator=gen))
            else:
                p.copy_(0.02 * torch.randn(p.shape, generator=gen))
    return w.cuda()


STAGE3 = {
    "dinov2-b-reg4-stride7": dict(ident="vit_base_patch14_reg4_dinov2.lvd142m", stride=7, depth=2, hw=(70, 84)),
    "clip-b16": dict(ident="vit_base_patch16_clip_224.openai", stride=16, depth=2, hw=(96, 112)),
    "mae-h14-hd80": dict(ident="vit_huge_patch14_224.mae", stride=14, depth=1, hw=(84, 98)),
    "vitg-swiglu": dict(ident="vit_giant_patch14_dinov2.lvd142m", stride=14, depth=2, hw=(70, 70)),
}


@pytest.mark.parametrize("case", list(STAGE3))
def test_stage3_bit_identical_with_and_without_checkpointing(det, case):
    from dvt import train_ops
    from dvt.optim import FusedAdamW
    c = STAGE3[case]
    w = _random_wrapper(c["ident"], c["stride"], c["depth"])
    sd = {k: v.detach().clone() for k, v in w.state_dict().items()}
    g = torch.Generator().manual_seed(2)
    imgs = [torch.randn(2, 3, *c["hw"], generator=g) for _ in range(10)]
    tgt_shape = w.get_intermediate_layers(imgs[0].cuda())[0].permute(0, 2, 3, 1).shape
    tgts = [torch.randn(tgt_shape, generator=g) for _ in range(10)]
    runs = []
    for ckpt in (False, False, True):
        w.load_state_dict(sd, strict=True)
        w.set_trainable(True)
        w.model.set_grad_checkpointing(ckpt)
        opt = FusedAdamW(w.parameters(), lr=1e-4, weight_decay=1e-5)
        logs = []
        for x, t in zip(imgs, tgts):
            pred = w.get_intermediate_layers(x.cuda())[0].permute(0, 2, 3, 1)
            loss, l2, cs = train_ops.denoise_loss(pred, t.cuda())
            opt.zero_grad()
            loss.backward()
            opt.step()
            logs.append(torch.stack([loss.detach(), l2.detach(), cs.detach()]))
        runs.append(_state(opt, logs))
        w.set_trainable(False)
    _dev_ok()
    _assert_same(runs[0], runs[1])
    _assert_same(runs[0], runs[2])


# ---------------------------------------------------------------------------------------------------------------------
# gradients against the fp32 oracle, in deterministic mode (the tolerances of the existing tests)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["reg4-stride7", "dino-s16-resampled"])
def test_stage3_gradients_match_oracle(det, case):
    import test_distill_gpu
    test_distill_gpu.test_vit_gradients_match_oracle(case)


@pytest.mark.parametrize("nb,hw_in", [(1, (5, 6)), (1, (7, 9))], ids=["one-block", "resampled-pe"])
def test_stage2_gradients_match_oracle(det, nb, hw_in):
    import test_train_gpu
    test_train_gpu.test_block_gradients_match_oracle(nb, hw_in)


# ---------------------------------------------------------------------------------------------------------------------
# command line
# ---------------------------------------------------------------------------------------------------------------------
def _ckpt_equal(a, b):
    assert a.keys() == b.keys() and a["step"] == b["step"]
    model_key = "model" if "model" in a else "denoiser"
    assert a[model_key].keys() == b[model_key].keys()
    for k in a[model_key]:
        assert torch.equal(a[model_key][k], b[model_key][k]), k
    sa, sb = a["optimizer"]["state"], b["optimizer"]["state"]
    assert sa.keys() == sb.keys() and len(sa) > 0
    for i in sa:
        for k in ("exp_avg", "exp_avg_sq", "step"):
            assert torch.equal(sa[i][k], sb[i][k]), (i, k)


def test_stage3_cli_deterministic(det, tmp_path, monkeypatch):
    from PIL import Image
    import dvt.models as DVT
    from dvt.models import vit_wrapper as VW
    sys.path.insert(0, ROOT)
    import main_distillation as M
    ident = "vit_small_patch14_reg4_dinov2.lvd142m"
    rs = np.random.RandomState(0)
    for i in range(8):
        d = tmp_path / "data" / f"class{i % 2}"
        d.mkdir(parents=True, exist_ok=True)
        Image.fromarray(rs.randint(0, 255, (70, 70, 3), dtype=np.uint8)).save(d / f"{i}.png")
    torch.manual_seed(0)
    vit = VW.B200VisionTransformer(ident, 14, VW.ARCHS[ident])
    wdir = tmp_path / "weights"
    wdir.mkdir()
    torch.save(vit.state_dict(), wdir / f"{ident}.pth")
    monkeypatch.setenv("DVT_WEIGHTS_DIR", str(wdir))
    den = DVT.Denoiser(9, 9, 384, vit=None, num_blocks=1)
    torch.save({"denoiser": den.state_dict(), "optimizer": {}, "step": 0}, tmp_path / "denoiser.pth")
    cks = []
    for run in ("a", "b"):
        argv = ["--model", ident, "--denoiser_ckpt", str(tmp_path / "denoiser.pth"), "--input_size", "70", "--stride_size", "7",
                "--data_root", str(tmp_path / "data"), "--batch_size", "4", "--num_iterations", "6", "--blr", "0.002",
                "--output_root", str(tmp_path / "work"), "--run_name", run, "--save_freq", "100", "--num_workers", "0",
                "--log_freq", "2", "--deterministic"]
        M.main(M.get_args(argv))
        cks.append(torch.load(str(tmp_path / "work" / "denosing-vit" / run / "checkpoints" / "latest.pth"), map_location="cpu"))
    _ckpt_equal(*cks)


def test_stage2_cli_deterministic(det, tmp_path):
    from argparse import Namespace
    sys.path.insert(0, ROOT)
    import main_denoiser as M
    from dvt.store import FeatureStoreWriter
    from dvt.utils import misc
    model = "vit_small_patch14_dinov2.lvd142m"
    h = w = 5
    data_root = str(tmp_path / "data") + "/"
    sargs = Namespace(data_root=data_root, save_root=str(tmp_path / "feats"), model=model)
    g = torch.Generator().manual_seed(0)
    wr = FeatureStoreWriter()
    rels = [f"img/{i}.jpg" for i in range(6)]
    for rel in rels:
        clean = torch.randn(h, w, 384, generator=g)
        wr.submit(*misc.feature_paths(sargs, os.path.join(data_root, rel)), clean + 0.3, clean[None])
    wr.close()
    lst = tmp_path / "list.txt"
    lst.write_text("".join(f"{r} 0\n" for r in rels))
    cks = []
    for run in ("a", "b"):
        argv = ["--model", model, "--input_size", "70", "--stride_size", "14", "--data_root", data_root, "--feat_root",
                f"{sargs.save_root}/denoised_features/{model}/", "--data_list_path", str(lst), "--batch_size", "4",
                "--num_iterations", "10", "--blr", "0.02", "--output_root", str(tmp_path / "work"), "--run_name", run,
                "--save_freq", "100", "--num_workers", "0", "--log_freq", "5", "--deterministic"]
        M.main(M.get_args(argv))
        cks.append(torch.load(str(tmp_path / "work" / "denosing-vit" / run / "checkpoints" / "latest.pth"), map_location="cpu"))
    _ckpt_equal(*cks)
