"""The fp64 training mirror (tests/train_oracle_fp64.py) and its error bound, proven on the host.

  * The math: with nothing rounded (fp64 saved tensors), every gradient of every node equals torch.autograd in fp64
    through oracle/vit.py / tests/vit_oracle_rope.py / oracle/denoiser.py to ~1e-12.
  * The bound admits an honest implementation: a CPU emulation of train_ops.py -- fp32 arithmetic, bf16 rounding exactly
    where the CUDA path rounds (d2, dhpre, d1, datt, dqkv, the RoPE backward's store, and P / dS inside a flash-style
    attention backward) -- stays within LAMBDA sqrt(var) with at least 2x of room, over every node option and 3 seeds.
  * Teeth: the simulated bugs the cosine tests cannot see, each built from the same emulation, are all rejected."""
import math

import pytest
import torch
import torch.nn.functional as F

import train_oracle_fp64 as T
import vit_oracle_rope as R
from oracle import vit as OV

# (C, heads, mlp hidden, swiglu, layerscale, rope, eps): every option of the block node at small widths
BLOCKS = {
    "denoiser": (128, 2, 512, False, False, False, 1e-6),
    "layerscale": (128, 2, 512, False, True, False, 1e-6),
    "hd80": (160, 2, 640, False, False, False, 1e-6),
    "swiglu": (128, 2, 512, True, True, False, 1e-6),
    "rope": (128, 2, 512, False, True, True, 1e-5),
}
B, H_GRID, W_GRID, PREFIX = 3, 4, 5, 5      # 3 images of 5 prefix + 20 patch rows: 75 token rows, a ragged last tile
ROOM = 0.5                                   # the honest worst ratio stays below this: >= 2x of room at LAMBDA


def b16(t):
    return t.bfloat16().float()


def _weights(name, seed):
    C, heads, hid, swiglu, ls, rope, eps = BLOCKS[name]
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s, std=1.0: torch.randn(*s, generator=g, dtype=torch.float64) * std   # noqa: E731
    fc2_in = hid // 2 if swiglu else hid
    w = dict(n1w=1 + rn(C, std=0.1), n1b=rn(C, std=0.1), wq=rn(3 * C, C, std=C ** -0.5), qkvb=rn(3 * C, std=0.3),
             wp=rn(C, C, std=0.5 * C ** -0.5), projb=rn(C, std=0.1), n2w=1 + rn(C, std=0.1), n2b=rn(C, std=0.1),
             w1=rn(hid, C, std=C ** -0.5), fc1b=rn(hid, std=0.1), w2=rn(C, fc2_in, std=0.5 * fc2_in ** -0.5),
             fc2b=rn(C, std=0.1), ls1=None, ls2=None)
    if ls:
        w["ls1"], w["ls2"] = 0.5 + torch.rand(C, generator=g, dtype=torch.float64), 0.5 + torch.rand(C, generator=g,
                                                                                                        dtype=torch.float64)
    if rope:
        w["qkvb"][C:2 * C] = 0
    # the GEMM weights the kernels read are bf16; LayerNorm / bias / LayerScale stay fp32
    for k in ("wq", "wp", "w1", "w2"):
        w[k] = b16(w[k]).double()
    for k in ("n1w", "n1b", "qkvb", "projb", "n2w", "n2b", "fc1b", "fc2b", "ls1", "ls2"):
        w[k] = None if w[k] is None else w[k].float().double()
    x0 = (rn(B * (PREFIX + H_GRID * W_GRID), C) * 2.0 + 0.3).float().double()
    dx2 = rn(*x0.shape).float().double()
    table = None
    if rope:
        cos, sin = R.rope_cos_sin(H_GRID, W_GRID)
        table = torch.cat([cos[:, :32], sin[:, :32]], 1)
    return w, x0, dx2, (None if table is None else (table, PREFIX)), heads, eps


# ------------------------------------------------------------------------------------------------ honest emulation
def _ln_bwd32(x, gamma, dy, eps):
    x, gamma, dy = x.float(), gamma.float(), dy.float()
    mu = x.mean(1, keepdim=True)
    rstd = ((x - mu).pow(2).mean(1, keepdim=True) + eps).rsqrt()
    xh = (x - mu) * rstd
    gd = dy * gamma
    dx = rstd * (gd - gd.mean(1, keepdim=True) - xh * (gd * xh).mean(1, keepdim=True))
    return dx, (dy * xh).sum(0), dy.sum(0)


def _flash_bwd32(qkv, out, dout, lse, batch, heads, block=64):
    """Key-block flash backward: fp32 P from the saved lse, bf16 P for dV, bf16 dS for dQ / dK, fp32 accumulators."""
    M, C3 = qkv.shape
    C = C3 // 3
    N, D = M // batch, C // heads
    t = qkv.float().view(batch, N, 3, heads, D).permute(2, 0, 3, 1, 4)
    q, k, v = t[0], t[1], t[2]
    hv = lambda a: a.float().view(batch, N, heads, D).permute(0, 2, 1, 3)    # noqa: E731
    dO, O = hv(dout), hv(out)
    delta = (dO * O).sum(-1, keepdim=True)
    scale = D ** -0.5
    dQ, dK, dV = torch.zeros_like(q), torch.zeros_like(k), torch.zeros_like(v)
    for j in range(0, N, block):
        kj, vj = k[:, :, j:j + block], v[:, :, j:j + block]
        s = (q @ kj.transpose(-1, -2)) * (scale * T.LOG2E)
        P = torch.exp2(s - lse.float()[..., None])
        dV[:, :, j:j + block] = b16(P).transpose(-1, -2) @ dO
        dP = dO @ vj.transpose(-1, -2)
        dS = b16(P * (dP - delta) * scale)
        dQ += dS @ kj
        dK[:, :, j:j + block] = dS.transpose(-1, -2) @ q
    back = lambda a: a.permute(0, 2, 1, 3).reshape(M, C)                   # noqa: E731
    return torch.cat([back(dQ), back(dK), back(dV)], 1)


def _rope_bwd32(dqkv, table, batch, prefix, heads, sign=-1.0):
    M, C3 = dqkv.shape
    t = dqkv.clone().view(batch, M // batch, 3, heads, C3 // 3 // heads)
    for j in range(2):
        t[:, prefix:, j] = T.rope_rot(t[:, prefix:, j], table[:, :32].float(), table[:, 32:].float(), sign)
    return b16(t.view(M, C3))


def emu_block_bwd(x0, acts, wts, dx2, *, heads, batch, eps, rope=None, bug=None, prefix=PREFIX):
    """train_ops._VitBlockFn.backward in fp32 with the CUDA path's bf16 roundings; `bug` plants one simulated defect."""
    a = {k: (None if v is None else v.float()) for k, v in acts.items()}
    w = {k: (None if v is None else v.float()) for k, v in wts.items()}
    x0, dx2 = x0.float(), dx2.float()
    M, C = x0.shape
    ntok = M // batch
    o = {}
    d2 = dx2 if w["ls2"] is None else dx2 * w["ls2"]
    o["fc2b"] = (d2 * w["ls2"]).sum(0) if bug == "ls_twice" else d2.sum(0)
    if w["ls2"] is not None:
        o["ls2"] = (dx2 * a["br2"]).sum(0)
    d2 = b16(d2)
    o["w2"] = d2.t() @ a["hid"]
    dh = d2 @ w["w2"]
    if 2 * w["w2"].shape[1] == w["w1"].shape[0]:
        Hh = w["w2"].shape[1]
        g, u = a["hpre"][:, :Hh], a["hpre"][:, Hh:]
        s = torch.sigmoid(g)
        dhpre = b16(torch.cat([dh * u * (s + g * s * (1 - s)), dh * g * s], 1))
    else:
        dhpre = b16(dh * T.gelu_grad(a["hpre"].double()).float())
    o["w1"] = dhpre[:-1].t() @ a["xn2"][:-1] if bug == "drop_row" else dhpre.t() @ a["xn2"]
    o["fc1b"] = dhpre.sum(0)
    dln, o["n2w"], o["n2b"] = _ln_bwd32(a["x1"], w["n2w"], dhpre @ w["w1"], eps)
    dx1 = dx2 + dln
    d1 = dx1 if w["ls1"] is None else dx1 * w["ls1"]
    o["projb"] = d1.sum(0)
    if w["ls1"] is not None:
        o["ls1"] = (dx1 * (a["br2"] if bug == "ls1_from_br2" else a["br1"])).sum(0)
    d1 = b16(d1)
    o["wp"] = d1.t() @ a["att"]
    datt = b16(d1 @ w["wp"])
    dqkv = b16(_flash_bwd32(a["qkv"], a["att"], datt, a["lse"], batch, heads))
    if bug == "head_swap":
        D = C // heads
        dqkv[:, D:2 * D] = dqkv[:, 0:D]
    if rope is not None:
        dqkv = _rope_bwd32(dqkv, rope[0], batch, rope[1], heads, sign=1.0 if bug == "rope_forward" else -1.0)
    o["wq"] = dqkv.t() @ a["xn1"]
    if bug == "colsum_no_prefix":
        o["qkvb"] = dqkv.view(batch, ntok, 3 * C)[:, prefix:].sum((0, 1))
    else:
        o["qkvb"] = dqkv.sum(0)
    if rope is not None and bug != "kbias_kept":
        o["qkvb"][C:2 * C] = 0
    dln, o["n1w"], o["n1b"] = _ln_bwd32(x0, w["n1w"], dqkv @ w["wq"], eps)
    o["x0"] = dx1 + dln
    return o


def _block_case(name, seed):
    w, x0, dx2, rope, heads, eps = _weights(name, seed)
    x2, acts = T.block_fwd64(x0, w, heads=heads, batch=B, eps=eps, rope=rope, round_to="bf16")
    return w, x0, dx2, rope, heads, eps, x2, acts


def _worst(got, ref):
    return {k: T.ratio(got[k], ref[k])[0] for k in ref}


# ------------------------------------------------------------------------------------------------ exact math
def _oracle_block_grads(name, w, x0, dx2, rope, heads, eps):
    C = x0.shape[1]
    hid = w["w1"].shape[0]
    cfg = OV.ViTConfig(C, 1, heads, 16, 224, hid, BLOCKS[name][3], w["ls1"] is not None, ln_eps=eps)
    names = {"n1w": "norm1.weight", "n1b": "norm1.bias", "wq": "attn.qkv.weight", "qkvb": "attn.qkv.bias",
             "wp": "attn.proj.weight", "projb": "attn.proj.bias", "ls1": "ls1.gamma", "n2w": "norm2.weight",
             "n2b": "norm2.bias", "w1": "mlp.fc1.weight", "fc1b": "mlp.fc1.bias", "w2": "mlp.fc2.weight",
             "fc2b": "mlp.fc2.bias", "ls2": "ls2.gamma"}
    p = {"blocks.0." + names[k]: v.clone().requires_grad_(True) for k, v in w.items() if v is not None}
    x = x0.clone().view(B, -1, C).requires_grad_(True)
    if rope is not None:
        cos, sin = R.rope_cos_sin(H_GRID, W_GRID)
        cfg = R.RopeViTConfig(C, 1, heads, 16, 224, hid, False, True, num_reg_tokens=PREFIX - 1, ln_eps=eps)
        y = R.block(x, p, 0, cfg, cos.double(), sin.double())
    else:
        y = OV.block(x, p, 0, cfg)
    y.backward(dx2.view(B, -1, C))
    out = {k: p["blocks.0." + names[k]].grad for k in w if w[k] is not None}
    out["x0"] = x.grad.view(-1, C)
    if rope is not None:
        out["qkvb"][C:2 * C] = 0
    return y.detach().reshape(-1, C), out


@pytest.mark.parametrize("name", list(BLOCKS))
def test_block_mirror_is_the_exact_gradient(name):
    w, x0, dx2, rope, heads, eps = _weights(name, 1)
    x2, acts = T.block_fwd64(x0, w, heads=heads, batch=B, eps=eps, rope=rope)
    y, ref = _oracle_block_grads(name, w, x0, dx2, rope, heads, eps)
    assert (x2 - y).abs().max().item() < 1e-12 * y.abs().max().item()
    got = T.block_bwd(x0, acts, w, T.exact(dx2), heads=heads, batch=B, eps=eps, rope=rope)
    assert set(got) == set(ref)
    for k, r in ref.items():
        err = (got[k].val - r).abs().max().item()
        assert err <= 1e-11 * r.abs().max().item() + 1e-300, f"{name} {k}: {err:.3g}"


def _embed_setup(seed, bias=True, pos=True, P=4, stride=3):
    g = torch.Generator().manual_seed(seed)
    C = 64
    img = torch.randn(B, 3, 13, 16, generator=g, dtype=torch.float64)
    pe_w = b16(torch.randn(C, 3, P, P, generator=g, dtype=torch.float64) * 0.2).double()
    pe_b = torch.randn(C, generator=g, dtype=torch.float64) if bias else None
    h, w = (13 - P) // stride + 1, (16 - P) // stride + 1
    pos_p = torch.randn(h * w, C, generator=g, dtype=torch.float64) if pos else None
    pre = torch.randn(PREFIX, C, generator=g, dtype=torch.float64)
    patches = b16(F.unfold(img, P, stride=stride).transpose(1, 2).reshape(-1, 3 * P * P)).double()
    dx0 = torch.randn(B * (PREFIX + h * w), C, generator=g, dtype=torch.float64).float().double()
    return img, pe_w, pe_b, pos_p, pre, patches, dx0, (h, w, C, P)


@pytest.mark.parametrize("bias,pos", [(True, True), (False, True), (True, False)])
def test_embed_mirror_is_the_exact_gradient(bias, pos):
    _, pe_w, pe_b, pos_p, pre, patches, dx0, (h, w, C, P) = _embed_setup(2, bias, pos)
    leaves = [t.clone().requires_grad_(True) if t is not None else None for t in (pe_w, pe_b, pos_p, pre)]
    tok = patches @ leaves[0].reshape(C, -1).t()
    if bias:
        tok = tok + leaves[1]
    tok = tok.view(B, h * w, C)
    if pos:
        tok = tok + leaves[2]
    y = torch.cat([leaves[3].expand(B, -1, -1), tok], 1).reshape(-1, C)
    y.backward(dx0)
    got = T.embed_bwd(patches, T.exact(dx0), batch=B, prefix=PREFIX, C=C, P=P)
    for k, leaf in zip(("pe_w", "pe_b", "pos", "prefix"), leaves):
        if leaf is not None:
            assert (got[k].val - leaf.grad).abs().max().item() <= 1e-12 * leaf.grad.abs().max().item(), k


def test_norm_loss_resample_mirrors_are_exact():
    g = torch.Generator().manual_seed(3)
    C, ntok = 64, PREFIX + 12
    x = (torch.randn(B * ntok, C, generator=g, dtype=torch.float64) * 3 + 1).requires_grad_(True)
    w = (1 + 0.2 * torch.randn(C, generator=g, dtype=torch.float64)).requires_grad_(True)
    b = torch.randn(C, generator=g, dtype=torch.float64).requires_grad_(True)
    dy = torch.randn(B * ntok, C, generator=g, dtype=torch.float64)
    F.layer_norm(x, (C,), w, b, 1e-5).backward(dy)
    got = T.layernorm_bwd(x.detach(), w.detach(), T.exact(dy), 1e-5)
    for k, r in (("x", x.grad), ("w", w.grad), ("b", b.grad)):
        assert (got[k].val - r).abs().max().item() <= 1e-12 * r.abs().max().item(), k
    for t in (x, w, b):
        t.grad = None
    dys = dy.view(B, ntok, C)[:, PREFIX:].reshape(-1, C)
    F.layer_norm(x, (C,), w, b, 1e-6).view(B, ntok, C)[:, PREFIX:].reshape(-1, C).backward(dys)
    got = T.norm_strip_bwd(x.detach(), w.detach(), T.exact(dys), ntok=ntok, prefix=PREFIX, eps=1e-6)
    for k, r in (("x", x.grad), ("w", w.grad), ("b", b.grad)):
        assert (got[k].val - r).abs().max().item() <= 1e-12 * r.abs().max().item(), k
    # loss
    p = torch.randn(2, 3, 4, C, generator=g, dtype=torch.float64).requires_grad_(True)
    t = torch.randn(2, 3, 4, C, generator=g, dtype=torch.float64)
    (F.mse_loss(p, t) + 1 - F.cosine_similarity(p, t, dim=-1).mean()).backward()
    assert (T.loss_bwd(p, t).val - p.grad.reshape(-1, C)).abs().max().item() <= 1e-13
    # resample
    gr = torch.randn(1, 8, 5, 6, generator=g, dtype=torch.float64).requires_grad_(True)
    do = torch.randn(1, 8, 7, 4, generator=g, dtype=torch.float64)
    F.interpolate(gr, size=(7, 4), mode="bicubic", antialias=True).backward(do)
    got = T.resample_bwd(T.exact(do), 5, 6)
    assert (got.val - gr.grad).abs().max().item() <= 1e-12 * gr.grad.abs().max().item()


# ------------------------------------------------------------------------------------------------ honest emulation
@pytest.mark.parametrize("name", list(BLOCKS))
def test_honest_block_emulation_within_bound(name):
    worst = {}
    for seed in (11, 12, 13):
        w, x0, dx2, rope, heads, eps, x2, acts = _block_case(name, seed)
        fwd = T.check_block_forward(x0, acts, w, x2, heads=heads, batch=B, eps=eps, rope=rope)
        assert max(fwd.values()) <= 1.0, fwd
        ref = T.block_bwd(x0, acts, w, T.exact(dx2), heads=heads, batch=B, eps=eps, rope=rope)
        emu = emu_block_bwd(x0, acts, w, dx2, heads=heads, batch=B, eps=eps, rope=rope)
        for k, r in _worst(emu, ref).items():
            worst[k] = max(worst.get(k, 0.0), r)
    print(f"\n{name}: worst |g - g64| / bound per tensor: " + " ".join(f"{k}={v:.3f}" for k, v in sorted(worst.items())))
    assert max(worst.values()) <= ROOM, worst


@pytest.mark.parametrize("bias,pos", [(True, True), (False, True), (True, False)], ids=["bias-pos", "no-bias", "no-pos"])
@pytest.mark.parametrize("seed", [4, 14, 24])
def test_honest_embed_within_bound(seed, bias, pos):
    _, pe_w, pe_b, pos_p, pre, patches, dx0, (h, w, C, P) = _embed_setup(seed, bias, pos)
    ref = T.embed_bwd(patches, T.exact(dx0), batch=B, prefix=PREFIX, C=C, P=P)
    emu = _emu_embed(patches, dx0, C, P)
    keep = ["pe_w", "prefix"] + (["pe_b"] if bias else []) + (["pos"] if pos else [])
    worst = _worst({k: emu[k] for k in keep}, {k: ref[k] for k in keep})
    print(f"\nembed seed {seed} bias {bias} pos {pos}: " + " ".join(f"{k}={v:.3f}" for k, v in sorted(worst.items())))
    assert max(worst.values()) <= ROOM, worst


@pytest.mark.parametrize("seed", [5, 15, 25])
def test_honest_norms_loss_resample_within_bound(seed):
    g = torch.Generator().manual_seed(seed)
    C, ntok = 64, PREFIX + 12
    x = (torch.randn(B * ntok, C, generator=g) * 3 + 1)
    wn = 1 + 0.2 * torch.randn(C, generator=g)
    worst = {}
    # norm_pre: LayerNorm over every token row (eps 1e-5, the CLIP towers)
    dy = torch.randn(B * ntok, C, generator=g)
    dx, dg, db = _ln_bwd32(x, wn, dy, 1e-5)
    ref = T.layernorm_bwd(x, wn, T.exact(dy), 1e-5)
    worst.update({f"norm_pre.{k}": v for k, v in _worst({"x": dx, "w": dg, "b": db}, ref).items()})
    # the final norm with the prefix strip
    dy = torch.randn(B * 12, C, generator=g)
    ref = T.norm_strip_bwd(x, wn, T.exact(dy), ntok=ntok, prefix=PREFIX, eps=1e-6)
    worst.update({f"norm.{k}": v for k, v in _worst(_emu_norm_strip(x, wn, dy, ntok, PREFIX, 1e-6), ref).items()})
    # the loss (torch's fp32 autograd of the same expression)
    p, t = torch.randn(40, C, generator=g), torch.randn(40, C, generator=g)
    pf = p.clone().requires_grad_(True)
    (F.mse_loss(pf, t) + 1 - F.cosine_similarity(pf, t, dim=-1).mean()).backward()
    worst["loss"] = T.ratio(pf.grad, T.loss_bwd(p, t))[0]
    # the resample backward, down and up (torch's fp32 backward)
    for (gh, gw), (oh, ow) in (((5, 6), (7, 4)), ((7, 7), (9, 8)), ((8, 8), (5, 13))):
        gr = torch.randn(1, 8, gh, gw, generator=g)
        do = torch.randn(1, 8, oh, ow, generator=g)
        grf = gr.clone().requires_grad_(True)
        F.interpolate(grf, size=(oh, ow), mode="bicubic", antialias=True).backward(do)
        worst[f"resample {gh}x{gw}->{oh}x{ow}"] = T.ratio(grf.grad, T.resample_bwd(T.exact(do), gh, gw))[0]
    print(f"\nseed {seed}: " + " ".join(f"{k}={v:.3f}" for k, v in worst.items()))
    assert max(worst.values()) <= ROOM, worst


def _emu_embed(patches, dx0, C, P, bug=None):
    t = dx0.float().view(B, -1, C)
    pat = t[:, PREFIX:]
    dpatch = b16(pat.reshape(-1, C))
    return {"pe_w": (dpatch.t() @ patches.float()).reshape(C, 3, P, P), "pe_b": pat.sum((0, 1)), "pos": pat.sum(0),
            "prefix": t[:1, :PREFIX].sum(0) if bug == "prefix_item0" else t[:, :PREFIX].sum(0)}


def _emu_norm_strip(x, wn, dy, ntok, prefix, eps, bug=None):
    C = x.shape[1]
    xb = x.float().view(B, ntok, C)
    dyb = dy.float().view(B, ntok - prefix, C)
    dx = torch.zeros_like(xb)
    dxk, dg, db = _ln_bwd32(xb[:, prefix:].reshape(-1, C), wn, dyb.reshape(-1, C), eps)
    dx[:, prefix:] = dxk.view(B, -1, C)
    if bug == "touch_prefix":   # the prefix rows normalised against the first patch row's gradient
        dxp, _, _ = _ln_bwd32(xb[:, :prefix].reshape(-1, C), wn, dyb[:, :1].expand(-1, prefix, -1).reshape(-1, C), eps)
        dx[:, :prefix] = dxp.view(B, prefix, C)
    return {"x": dx.view(-1, C), "w": dg, "b": db}


# ------------------------------------------------------------------------------------------------ teeth
BLOCK_BUGS = [("drop_row", "layerscale", "w1"), ("head_swap", "hd80", "wq"), ("colsum_no_prefix", "layerscale", "qkvb"),
              ("ls1_from_br2", "swiglu", "ls1"), ("rope_forward", "rope", "wq"), ("ls_twice", "layerscale", "fc2b"),
              ("kbias_kept", "rope", "qkvb")]


@pytest.mark.parametrize("bug,name,tensor", BLOCK_BUGS, ids=[b[0] for b in BLOCK_BUGS])
def test_simulated_block_bug_is_rejected(bug, name, tensor):
    w, x0, dx2, rope, heads, eps, x2, acts = _block_case(name, 21)
    ref = T.block_bwd(x0, acts, w, T.exact(dx2), heads=heads, batch=B, eps=eps, rope=rope)
    emu = emu_block_bwd(x0, acts, w, dx2, heads=heads, batch=B, eps=eps, rope=rope, bug=bug)
    r = _worst(emu, ref)
    assert r[tensor] > 1.0, f"{bug}: {tensor} ratio {r[tensor]:.3g} not rejected"


def test_simulated_dprefix_of_item0_only_is_rejected():
    _, _, _, _, _, patches, dx0, (h, w, C, P) = _embed_setup(6)
    ref = T.embed_bwd(patches, T.exact(dx0), batch=B, prefix=PREFIX, C=C, P=P)
    assert _worst(_emu_embed(patches, dx0, C, P, bug="prefix_item0"), ref)["prefix"] > 1.0


def test_simulated_final_norm_touching_prefix_rows_is_rejected():
    g = torch.Generator().manual_seed(7)
    C, ntok = 64, PREFIX + 12
    x = torch.randn(B * ntok, C, generator=g) * 3 + 1
    wn = 1 + 0.2 * torch.randn(C, generator=g)
    dy = torch.randn(B * 12, C, generator=g)
    ref = T.norm_strip_bwd(x, wn, T.exact(dy), ntok=ntok, prefix=PREFIX, eps=1e-6)
    assert _worst(_emu_norm_strip(x, wn, dy, ntok, PREFIX, 1e-6, bug="touch_prefix"), ref)["x"] > 1.0
