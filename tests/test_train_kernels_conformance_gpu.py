"""Conformance of the bandwidth-bound training and token-assembly kernels against fp64 references, at the shapes where
they go wrong: every NV / KV register width on both sides of its boundary, partial float4 lanes, row pitches wider than
the row, grid-stride loops and the chunk edges of the two-level reductions.

Every reference is fp64 computed from the exact fp32 / bf16 values the kernel reads.  u = 2^-24 is the fp32 unit
roundoff.  Each bound is per element and scaled by an absolute quantity, so that cancellation cannot hide an error.

LayerNorm forward (warp per row: each lane adds its 4*NV elements in pairs, then a 5-level shuffle tree; the centred
squares the same way; rsqrtf).  With sigma_e = sqrt(var + eps), m = max|x| of the row and xhat = (x - mean) / sigma_e:
the mean is off by at most (2 NV + 7) u m <= 40 u m, so x - mean is off by 40 u m + u |x - mean|; the variance is centred,
so the mean error enters it only to second order, and its own sum and rsqrtf add ~45 u relative to rstd.  Hence
|dxhat| <= 40 u m / sigma_e + 50 u |xhat| < 2^-17 (1 + |xhat|)(1 + m / sigma_e) (a factor ~2.5 of room), and
  |y - ref| <= 2^-17 |gamma| (1 + |xhat|)(1 + m / sigma_e) + 2^-23 (|ref| + |beta|)   (the last term: the final FMA and add).
  bf16 output: equal to RN-bf16 of the fp32 output, bit for bit.

LayerNorm backward.  g = dy * gamma; dx = rstd (g - mean(g) - xhat mean(g xhat)).  The xhat error above enters mean(g xhat)
as mean|g| dxhat, which the xhat factor multiplies again; the sums add <= 40 u of their absolute sums:
  |dx - ref| <= 2^-15 rstd (|g| + mean|g| (1 + |xhat|) + |xhat| mean|g xhat|)(1 + m / sigma_e) + 2^-23 |ref|
(2^-15 = 512 u: chains of ~40 additions, times the (1 + |xhat|) and rstd factors, with a factor ~2 of room).
dgamma = sum_r dy xhat and dbeta = sum_r dy are sums along chains of at most L = ceil(rows / (8 blocks)) + 8 + blocks + 2
additions (a warp's rows in order, the 8 warps of a CTA, the CTAs):
  |dgamma - ref| <= L u sum_r |dy xhat| + sum_r |dy| 2^-17 (1 + |xhat|)(1 + m / sigma_e),  |dbeta - ref| <= L u sum_r |dy|.

Column sums (dvt_colsum, dvt_colsum_ordered, the dbias / dgamma / dpos / dprefix sums of the LayerScale and token-assembly
backward): |out - ref| <= (L + 1) u sum_r |term|, with L the longest addition chain of the kernel's own grid (computed
below from the launcher's formulas).  dbranch and dpatch are RN-bf16 of the fp32 product gamma * dx (of dx0): exact.

Token assembly (dvt_vit_embed_fwd, GEMM with the OUT_F32_REMAP epilogue): as in test_gemm_conformance_gpu.py,
  |out - ref| <= 2^-18 P + 2^-23 |ref|,  P = |patches| |W|^T + |bias| + |pos|;  prefix rows equal prefix_rows exactly.

Denoising loss (dpred = k_mse (p - t) + k_t t + k_p p per element, the row dot products and norms as in LayerNorm):
  |dpred - ref| <= 2^-17 s (2 |p - t| / (rows C) + (|t| / (|p| |t|) + |p| / |p|^2) / rows) + 2^-23 |ref|
(norms clamped at 1e-8 as torch does; s = grad_scale).  The loss terms are sums of non-negative terms: the mse is within
(L + 4) u of its value, the cosine term within (L + 4 NV + 24) u (|cos term| + 1) (each row's cosine is within ~(4 NV + 20) u
absolutely, by Cauchy-Schwarz).  L = in-row chain + rows per warp + 8 + CTAs.

AdamW: one step at a time against torch.optim.AdamW(foreach=False) in fp64, from the kernel's own fp32 state.  The kernel
rounds beta1, beta2, eps, 1 - lr wd, lr / bc1 and 1 / sqrt(bc2) to fp32 (beta rounded by <= 2^-25 absolutely, which is
~2^-15 relative to 1 - beta2):
  |m - ref| <= 2^-22 (b1 |m0| + (1 - b1) |g|) + 2^-24 (|m0| + |g|),  |v - ref| likewise with v0 and g^2,
  |p - ref| <= 2^-22 |p0| + s dm / D + U dv / (2 v) + 2^-20 U,
D = sqrt(v) / sqrt(bc2) + eps, U = s |m| / D the update, s = lr / bc1.  A zero gradient over a zero state leaves
exactly RN(p * RN(1 - lr wd)).

Resample backward (two passes of in-order FMA chains of lengths h and w): |dgrid - ref| <= (h + w + 4) u |Wh|^T |dout| |Ww|.
im2col: equal to F.unfold of the bf16-rounded input, bit for bit, with zero K padding.
Segmentation loss: the fp64-autograd tolerance of test_dense_eval_gpu.py (1e-5 relative), at every KV width.

The bounds' teeth are shown on the host (no GPU needed): simulated wrong results built from the same inputs must be
rejected, and an fp32 evaluation of the right formula must pass."""
import math

import pytest
import torch
import torch.nn.functional as F

U = 2.0 ** -24
BF16, F32 = 0, 1
SENT = -7777.0                     # sentinel of the output padding: any store there changes it
C_SET = (4, 124, 128, 132, 384, 388, 768, 772, 1024, 1028, 1280, 1536, 1540, 2044, 2048)   # NV = 3, 6, 8, 12, 16 and tails
NSM_HOST = 132                     # the H100 SXM's SM count, for the host self-checks


def _nv(C):
    nv = (C // 4 + 31) // 32
    return 3 if nv <= 3 else 6 if nv <= 6 else 8 if nv <= 8 else 12 if nv <= 12 else 16


def ratio(out, ref, bound):
    """max |out - ref| / bound over elements (NaN in out counts as infinitely far)."""
    err = (out.double() - ref.double()).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    return (err / (bound.double() + 1e-300)).max().item()


def assert_within(out, ref, bound, what):
    r = ratio(out, ref, bound)
    assert r <= 1.0, f"{what}: error {r:.3g} x the bound"


# ------------------------------------------------------------------------------------------------ inputs
FAMILIES = ("gauss", "offset", "tiny_sigma", "constant", "nan")


def ln_rows(rows, C, seed, families=FAMILIES):
    """fp32 rows cycling through the row families: Gaussian; offset 1e3 with sigma 1; sigma 1e-3 (sigma^2 = eps); constant;
    one NaN element."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, C, generator=g, dtype=torch.float64)
    for r in range(rows):
        f = families[r % len(families)]
        if f == "offset":
            x[r] += 1e3
        elif f == "tiny_sigma":
            x[r] *= 1e-3
        elif f == "constant":
            x[r] = 3.7
        elif f == "nan":
            x[r, (r * 7) % C] = math.nan
    return x.float()


def ln_params(C, seed):
    g = torch.Generator().manual_seed(seed)
    return ((1 + 0.1 * torch.randn(C, generator=g, dtype=torch.float64)).float(),
            (0.1 * torch.randn(C, generator=g, dtype=torch.float64)).float())


# ------------------------------------------------------------------------------------------------ references and bounds
def ln_stats(x, eps):
    x = x.double()
    mean = x.mean(1, keepdim=True)
    var = ((x - mean) ** 2).mean(1, keepdim=True)
    sig = (var + eps).sqrt()
    m = x.abs().amax(1, keepdim=True)
    return (x - mean) / sig, sig, m


def ln_fwd_ref(x, gamma, beta, eps):
    xhat, sig, m = ln_stats(x, eps)
    g, b = gamma.double(), beta.double()
    ref = xhat * g + b
    bound = 2.0 ** -17 * g.abs() * (1 + xhat.abs()) * (1 + m / sig) + 2.0 ** -23 * (ref.abs() + b.abs())
    return ref, bound


def ln_bwd_ref(x, gamma, dy, eps):
    """(dx, dgamma, dbeta) in fp64 autograd, and the per-element dx bound and the per-row dgamma error term."""
    x64 = x.double().requires_grad_(True)
    g64, b64 = gamma.double().requires_grad_(True), torch.zeros_like(gamma, dtype=torch.float64).requires_grad_(True)
    y = F.layer_norm(x64, (x.shape[1],), g64, b64, eps)
    y.backward(dy.double())
    xhat, sig, m = ln_stats(x, eps)
    gg = dy.double() * gamma.double()
    amp = 1 + m / sig
    dx_bound = 2.0 ** -15 / sig * (gg.abs() + gg.abs().mean(1, keepdim=True) * (1 + xhat.abs())
                                   + xhat.abs() * (gg * xhat).abs().mean(1, keepdim=True)) * amp
    dxhat = 2.0 ** -17 * (1 + xhat.abs()) * amp
    return x64.grad, g64.grad, b64.grad, dx_bound, xhat, dxhat


def ln_bwd_param_bounds(dy, xhat, dxhat, L):
    dy = dy.double()
    return (L * U * (dy * xhat).abs().sum(0) + (dy.abs() * dxhat).sum(0), L * U * dy.abs().sum(0))


def ln_bwd_chain(rows, blocks):
    return -(-rows // (8 * blocks)) + 8 + blocks + 2


def loss_ref(pred, tgt, grad_scale):
    p = pred.double().requires_grad_(True)
    t = tgt.double()
    l2 = F.mse_loss(p, t)
    cos = 1 - F.cosine_similarity(p, t, dim=-1).mean()
    (l2 + cos).backward()
    return l2.item(), cos.item(), p.grad * grad_scale


def loss_dpred_bound(pred, tgt, grad_scale):
    p, t = pred.double(), tgt.double()
    rows, C = p.shape
    np_ = p.norm(dim=1, keepdim=True).clamp_min(1e-8)
    nt = t.norm(dim=1, keepdim=True).clamp_min(1e-8)
    return 2.0 ** -17 * grad_scale * (2 * (p - t).abs() / (rows * C) + (t.abs() / (np_ * nt) + p.abs() / np_ ** 2) / rows)


def loss_value_bounds(l2, cos, rows, C, blocks):
    nv = _nv(C)
    L = (2 * nv + 7) + -(-rows // (blocks * 8)) + 8 + blocks + 2
    return (L + 4) * U * abs(l2), (L + 4 * nv + 24) * U * (abs(cos) + 1)


ADAM = dict(lr=1e-3, b1=0.9, b2=0.999, eps=1e-8)


def adamw_ref(p, g, m, v, step, wd, lr=ADAM["lr"], b1=ADAM["b1"], b2=ADAM["b2"], eps=ADAM["eps"]):
    """One torch.optim.AdamW step in fp64 from the given fp32 state (step counts from 1), with the bounds."""
    P = torch.nn.Parameter(p.double().clone())
    P.grad = g.double().clone()
    opt = torch.optim.AdamW([P], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wd, foreach=False)
    opt.state[P] = {"step": torch.tensor(float(step - 1)), "exp_avg": m.double().clone(),
                    "exp_avg_sq": v.double().clone()}
    opt.step()
    st = opt.state[P]
    m1, v1 = st["exp_avg"], st["exp_avg_sq"]
    g64, m0, v0 = g.double(), m.double(), v.double()
    dm = 2.0 ** -22 * (b1 * m0.abs() + (1 - b1) * g64.abs()) + U * (m0.abs() + g64.abs())
    dv = 2.0 ** -22 * (b2 * v0 + (1 - b2) * g64 ** 2) + U * (v0 + g64 ** 2)
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    s = lr / bc1
    D = v1.sqrt() / math.sqrt(bc2) + eps
    upd = s * m1.abs() / D
    dp = 2.0 ** -22 * p.double().abs() + s * dm / D + upd * dv / (2 * v1.clamp_min(1e-300)) + 2.0 ** -20 * upd
    return P.detach(), m1, v1, dp, dm, dv


# ------------------------------------------------------------------------------------------------ host self-checks
def _ln_fwd_fp32(x, gamma, beta, eps, *, one_pass=False, eps_outside=False, drop_last4=False):
    """fp32 evaluation of LayerNorm, right or with a simulated defect."""
    xs = x[:, :-4] if drop_last4 else x
    C = xs.shape[1]
    mean = xs.sum(1, keepdim=True) / C
    if one_pass:
        var = (xs * xs).sum(1, keepdim=True) / C - mean * mean
    else:
        var = ((xs - mean) ** 2).sum(1, keepdim=True) / C
    rstd = (torch.rsqrt(var) + eps) if eps_outside else torch.rsqrt(var + eps)
    return (x - mean) * rstd * gamma + beta


def test_selfcheck_layernorm_bounds():
    C, eps = 768, 1e-6
    gamma, beta = ln_params(C, 1)
    for fam, defect in (("offset", "one_pass"), ("tiny_sigma", "eps_outside"), ("gauss", "drop_last4"),
                        ("offset", "drop_last4")):
        x = ln_rows(16, C, 2, families=(fam,))
        ref, bound = ln_fwd_ref(x, gamma, beta, eps)
        assert ratio(_ln_fwd_fp32(x, gamma, beta, eps), ref, bound) <= 1.0, fam
        assert ratio(_ln_fwd_fp32(x, gamma, beta, eps, **{defect: True}), ref, bound) > 1.0, (fam, defect)


def _ln_bwd_fp32(x, gamma, dy, eps, *, no_mgx=False):
    C = x.shape[1]
    mean = x.sum(1, keepdim=True) / C
    rstd = torch.rsqrt(((x - mean) ** 2).sum(1, keepdim=True) / C + eps)
    xhat = (x - mean) * rstd
    g = dy * gamma
    mg = g.sum(1, keepdim=True) / C
    mgx = (g * xhat).sum(1, keepdim=True) / C
    return rstd * (g - mg - (0 if no_mgx else xhat * mgx)), xhat


def test_selfcheck_layernorm_bwd_bounds():
    C, eps = 384, 1e-6
    gamma, _ = ln_params(C, 3)
    for fam in ("gauss", "offset", "tiny_sigma"):
        x = ln_rows(64, C, 4, families=(fam,))
        dy = torch.randn(64, C, generator=torch.Generator().manual_seed(5))
        dx_ref, _, _, bound, _, _ = ln_bwd_ref(x, gamma, dy, eps)
        good, _ = _ln_bwd_fp32(x, gamma, dy, eps)
        assert ratio(good, dx_ref, bound) <= 1.0, fam
        if fam == "gauss":
            bad, _ = _ln_bwd_fp32(x, gamma, dy, eps, no_mgx=True)
            assert ratio(bad, dx_ref, bound) > 1.0


def test_selfcheck_dgamma_rejects_a_missing_cta_partial():
    rows, C, eps = 1000, 384, 1e-6
    blocks = min(NSM_HOST, (rows + 7) // 8)
    gamma, _ = ln_params(C, 6)
    x = ln_rows(rows, C, 7, families=("gauss",))
    dy = torch.randn(rows, C, generator=torch.Generator().manual_seed(8))
    _, dg_ref, db_ref, _, xhat, dxhat = ln_bwd_ref(x, gamma, dy, eps)
    bg, bb = ln_bwd_param_bounds(dy, xhat, dxhat, ln_bwd_chain(rows, blocks))
    _, xh32 = _ln_bwd_fp32(x, gamma, dy, eps)
    assert ratio((dy * xh32).sum(0), dg_ref, bg) <= 1.0 and ratio(dy.sum(0), db_ref, bb) <= 1.0
    keep = torch.tensor([(r // 8) % blocks != 0 for r in range(rows)])   # CTA 0's warps own rows 8 k blocks + 0..7
    assert ratio((dy * xh32)[keep].sum(0), dg_ref, bg) > 1.0
    assert ratio(dy[keep].sum(0), db_ref, bb) > 1.0


def _adamw_fp32(p, g, m, v, step, wd, *, no_bc2=False, eps_inside=False, lr=ADAM["lr"], b1=ADAM["b1"], b2=ADAM["b2"],
                eps=ADAM["eps"]):
    f = lambda a: torch.tensor(a, dtype=torch.float32)   # noqa: E731
    bc1, bc2 = 1 - b1 ** step, 1 - b2 ** step
    b1f, b2f = f(b1), f(b2)
    p = p * f(1 - lr * wd)
    m = b1f * m + (1 - b1f) * g
    v = b2f * v + (1 - b2f) * g * g
    if eps_inside:
        den = torch.sqrt(v / f(bc2) + f(eps))
    else:
        den = torch.sqrt(v) * (f(1.0) if no_bc2 else f(1 / math.sqrt(bc2))) + f(eps)
    return p - f(lr / bc1) * m / den, m, v


def test_selfcheck_adamw_bounds():
    gen = torch.Generator().manual_seed(9)
    n = 4096
    p, g = torch.randn(n, generator=gen), torch.randn(n, generator=gen) * 1e-2
    m, v = torch.randn(n, generator=gen) * 1e-3, torch.rand(n, generator=gen) * 1e-4
    for step in (2, 10):
        pr, mr, vr, dp, dm, dv = adamw_ref(p, g, m, v, step, 0.05)
        p1, m1, v1 = _adamw_fp32(p, g, m, v, step, 0.05)
        assert ratio(p1, pr, dp) <= 1 and ratio(m1, mr, dm) <= 1 and ratio(v1, vr, dv) <= 1
        assert ratio(_adamw_fp32(p, g, m, v, step, 0.05, no_bc2=True)[0], pr, dp) > 1.0
        assert ratio(_adamw_fp32(p, g, m, v, step, 0.05, eps_inside=True)[0], pr, dp) > 1.0


def _loss_dpred_fp32(p, t, grad_scale, *, no_cos_term=False):
    rows, C = p.shape
    np_ = p.norm(dim=1, keepdim=True).clamp_min(1e-8)
    nt = t.norm(dim=1, keepdim=True).clamp_min(1e-8)
    cos = (p * t).sum(1, keepdim=True) / (np_ * nt)
    d = 2 * (p - t) / (rows * C) - t / (np_ * nt) / rows
    if not no_cos_term:
        d = d + cos * p / (np_ * np_) / rows
    return d * grad_scale


def test_selfcheck_loss_gradient_bound():
    gen = torch.Generator().manual_seed(10)
    t = torch.randn(64, 384, generator=gen)
    p = 0.7 * t + 0.5 * torch.randn(64, 384, generator=gen)       # cosine ~0.8: the cos p / |p|^2 term matters
    p[3] = 0
    _, _, ref = loss_ref(p, t, 2.0)
    bound = loss_dpred_bound(p, t, 2.0) + 2.0 ** -23 * ref.abs()
    assert ratio(_loss_dpred_fp32(p, t, 2.0), ref, bound) <= 1.0
    assert ratio(_loss_dpred_fp32(p, t, 2.0, no_cos_term=True), ref, bound) > 1.0


# ------------------------------------------------------------------------------------------------ GPU helpers
@pytest.fixture(scope="module")
def L():
    from dvt import _lib
    return _lib


def _nsm():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ptr(t, offset_elems=0):
    from ctypes import c_void_p
    return None if t is None else c_void_p(t.data_ptr() + offset_elems * t.element_size())


def _st():
    from dvt._lib import cur_stream
    return cur_stream()


def _pitched(a, ld, fill=math.nan):
    """a [rows, C] placed in the first C columns of a [rows, ld] buffer whose other columns hold `fill`."""
    buf = torch.full((a.shape[0], ld), fill, dtype=a.dtype, device="cuda")
    buf[:, :a.shape[1]] = a.cuda()
    return buf


# ------------------------------------------------------------------------------------------------ LayerNorm forward
def _ln_fwd(L, x_buf, gamma, beta, rows, C, eps, y_dtype, out_rows, ldy, in_group=1, skip=0, extra_rows=3):
    """Runs dvt_layernorm into a [out_rows + extra_rows, ldy] buffer: NaN where the output goes, SENT elsewhere.  Checks that
    nothing outside [out_rows, C] changed and returns the [out_rows, C] output."""
    dt = torch.bfloat16 if y_dtype == BF16 else torch.float32
    y = torch.full((out_rows + extra_rows, ldy), SENT, dtype=dt, device="cuda")
    y[:out_rows, :C] = math.nan
    L.check(L.lib().dvt_layernorm(_ptr(x_buf), x_buf.stride(0), _ptr(gamma), _ptr(beta), _ptr(y), ldy, y_dtype, rows, C, eps,
                                  in_group, skip, _st()), "dvt_layernorm")
    torch.cuda.synchronize()
    assert bool((y[:, C:] == SENT).all()) and bool((y[out_rows:] == SENT).all()), "store outside the output"
    return y[:out_rows, :C]


@pytest.mark.gpu
@pytest.mark.parametrize("C", C_SET)
def test_layernorm_fwd(L, C):
    eps = 1e-6
    gamma, beta = ln_params(C, C)
    x = ln_rows(257, C, C + 1)
    x_buf = _pitched(x, C + 12)
    g, b = gamma.cuda(), beta.cuda()
    nan_rows = torch.tensor([FAMILIES[r % 5] == "nan" for r in range(257)])
    for rows in (1, 7, 8, 9, 257):
        ref, bound = ln_fwd_ref(x[:rows], gamma, beta, eps)
        y = _ln_fwd(L, x_buf, g, b, rows, C, eps, F32, rows, C + 8).cpu()
        nr = nan_rows[:rows]
        assert bool(torch.isnan(y[nr]).all()), "a NaN input row must give a NaN row"
        if (~nr).any():
            assert_within(y[~nr], ref[~nr], bound[~nr], f"LN fwd C={C} rows={rows}")
        yb = _ln_fwd(L, x_buf, g, b, rows, C, eps, BF16, rows, C + 4).cpu()
        assert torch.equal(yb.view(torch.int16)[~nr], y.bfloat16().view(torch.int16)[~nr]), "bf16 != RN-bf16(f32)"
        assert bool(torch.isnan(yb[nr]).all())
    # prefix strip: the in_group / skip output is the plain output's kept rows, bit for bit (rows = 250: 25 groups of 10)
    rows, grp, skip = 250, 10, 3
    y = _ln_fwd(L, x_buf, g, b, rows, C, eps, F32, rows, C)
    ys = _ln_fwd(L, x_buf, g, b, rows, C, eps, F32, rows // grp * (grp - skip), C + 4, in_group=grp, skip=skip)
    keep = torch.tensor([r % grp >= skip for r in range(rows)], device="cuda")
    assert torch.equal(ys.view(torch.int32), y[keep].contiguous().view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("C", [384, 1280, 2048])
def test_layernorm_fwd_grid_stride(L, C):
    """More rows than one full wave of warps (occupancy x #SM x 8): the grid-stride loop runs several times."""
    eps, rows = 1e-6, 8 * 16 * _nsm() * 2 + 37
    gamma, beta = ln_params(C, 3 * C)
    x = ln_rows(rows, C, C + 2, families=("gauss", "offset", "tiny_sigma"))
    ref, bound = ln_fwd_ref(x, gamma, beta, eps)
    y = _ln_fwd(L, x.cuda(), gamma.cuda(), beta.cuda(), rows, C, eps, F32, rows, C).cpu()
    assert_within(y, ref, bound, f"LN fwd grid-stride C={C}")


# ------------------------------------------------------------------------------------------------ LayerNorm backward
def _ln_bwd_case(L, x, gamma, dy, eps, acc0, grouped, in_group=1, skip=0):
    rows, C = x.shape
    xd, gd, dyd = x.cuda(), gamma.cuda(), dy.cuda()
    acc = acc0.clone().cuda()
    if grouped:
        dg, db = torch.full((C,), math.nan, device="cuda"), torch.full((C,), math.nan, device="cuda")
        ws = torch.empty(256 * C, device="cuda")
        L.check(L.lib().dvt_layernorm_bwd_grouped(_ptr(xd), _ptr(gd), _ptr(dyd), _ptr(acc), _ptr(dg), _ptr(db), _ptr(ws), rows,
                                                  C, eps, in_group, skip, _st()), "dvt_layernorm_bwd_grouped")
    else:
        dg, db = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
        L.check(L.lib().dvt_layernorm_bwd(_ptr(xd), _ptr(gd), _ptr(dyd), _ptr(acc), _ptr(dg), _ptr(db), rows, C, eps, _st()),
                "dvt_layernorm_bwd")
    torch.cuda.synchronize()
    return acc.cpu(), dg.cpu(), db.cpu()


def _check_ln_bwd(x, gamma, dy, eps, acc0, acc, dg, db, blocks, what):
    dx_ref, dg_ref, db_ref, dx_bound, xhat, dxhat = ln_bwd_ref(x, gamma, dy, eps)
    ref = acc0.double() + dx_ref
    assert_within(acc, ref, dx_bound + 2.0 ** -23 * ref.abs(), f"{what} dx")
    bg, bb = ln_bwd_param_bounds(dy, xhat, dxhat, ln_bwd_chain(x.shape[0], blocks))
    assert_within(dg, dg_ref, bg, f"{what} dgamma")
    assert_within(db, db_ref, bb, f"{what} dbeta")


BWD_FAMILIES = ("gauss", "offset", "tiny_sigma", "constant")


@pytest.mark.gpu
@pytest.mark.parametrize("C", C_SET)
def test_layernorm_bwd(L, C):
    eps, rows = 1e-6, 257
    gamma, _ = ln_params(C, 5 * C)
    x = ln_rows(rows, C, C + 3, families=BWD_FAMILIES)
    gen = torch.Generator().manual_seed(C + 4)
    dy = torch.randn(rows, C, generator=gen)
    acc0 = torch.randn(rows, C, generator=gen)                       # dx_accum starts nonzero
    plain = _ln_bwd_case(L, x, gamma, dy, eps, acc0, False)
    _check_ln_bwd(x, gamma, dy, eps, acc0, *plain, min(_nsm(), (rows + 7) // 8), f"LN bwd C={C}")
    grouped = _ln_bwd_case(L, x, gamma, dy, eps, acc0, True)
    _check_ln_bwd(x, gamma, dy, eps, acc0, *grouped, min(128, (rows + 7) // 8), f"LN bwd grouped C={C}")
    assert torch.equal(plain[0].view(torch.int32), grouped[0].view(torch.int32)), \
        "dvt_layernorm_bwd and dvt_layernorm_bwd_grouped(1, 0) must give the same dx bits"


@pytest.mark.gpu
@pytest.mark.parametrize("C", [384, 1280])
def test_layernorm_bwd_grid_edges(L, C):
    """Row counts around min(#SM, ceil(rows / 8)) (plain) and min(128, ceil(rows / 8)) (grouped), and a grid-stride case."""
    eps = 1e-6
    gamma, _ = ln_params(C, 7 * C)
    nsm = _nsm()
    for rows in sorted({1, 8 * nsm - 1, 8 * nsm + 1, 1023, 1025, 20000}):
        x = ln_rows(rows, C, rows + C, families=("gauss", "offset"))
        gen = torch.Generator().manual_seed(rows)
        dy, acc0 = torch.randn(rows, C, generator=gen), torch.randn(rows, C, generator=gen)
        _check_ln_bwd(x, gamma, dy, eps, acc0, *_ln_bwd_case(L, x, gamma, dy, eps, acc0, False), min(nsm, (rows + 7) // 8),
                      f"LN bwd rows={rows}")
        _check_ln_bwd(x, gamma, dy, eps, acc0, *_ln_bwd_case(L, x, gamma, dy, eps, acc0, True), min(128, (rows + 7) // 8),
                      f"LN bwd grouped rows={rows}")


@pytest.mark.gpu
@pytest.mark.parametrize("C", [132, 1028])
def test_layernorm_bwd_grouped_skip(L, C):
    """The prefix-strip form: dy holds the kept rows only, skipped rows of dx_accum stay bit-identical."""
    eps, grp, skip, ngroups = 1e-6, 10, 3, 151
    rows = grp * ngroups
    gamma, _ = ln_params(C, 11 * C)
    x = ln_rows(rows, C, C + 5, families=BWD_FAMILIES)
    keep = torch.tensor([r % grp >= skip for r in range(rows)])
    gen = torch.Generator().manual_seed(C + 6)
    dy_full = torch.randn(rows, C, generator=gen)
    dy_full[~keep] = 0
    acc0 = torch.randn(rows, C, generator=gen)
    acc, dg, db = _ln_bwd_case(L, x, gamma, dy_full[keep].contiguous(), eps, acc0, True, grp, skip)
    assert torch.equal(acc[~keep].view(torch.int32), acc0[~keep].view(torch.int32)), "a skipped row was written"
    out_rows = ngroups * (grp - skip)
    dx_ref, dg_ref, db_ref, dx_bound, xhat, dxhat = ln_bwd_ref(x[keep], gamma, dy_full[keep], eps)
    ref = acc0[keep].double() + dx_ref
    assert_within(acc[keep], ref, dx_bound + 2.0 ** -23 * ref.abs(), "grouped dx")
    bg, bb = ln_bwd_param_bounds(dy_full[keep], xhat, dxhat, ln_bwd_chain(out_rows, min(128, (out_rows + 7) // 8)))
    assert_within(dg, dg_ref, bg, "grouped dgamma")
    assert_within(db, db_ref, bb, "grouped dbeta")


# ------------------------------------------------------------------------------------------------ column sums
def _colsum_chain_atomic(rows, cols, bf16, nsm):
    gx = -(-cols // (64 if bf16 else 32))
    gy = max(1, min(-(-rows // 64), -(-(nsm * 4) // gx)))
    return -(-(-(-rows // gy)) // 8) + 8 + gy + 1


def _det_chunks(rows):
    return max(1, min(128, -(-rows // 64)))


def _chain_ordered(rows):
    ch = _det_chunks(rows)
    return -(-(-(-rows // ch)) // 8) + 8 + ch + 1


def _colsum_input(rows, cols, bf16, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(rows, cols, generator=g) + 0.5                 # a nonzero mean: a dropped chunk shows
    return a.bfloat16() if bf16 else a


@pytest.mark.gpu
@pytest.mark.parametrize("bf16", [False, True], ids=["f32", "bf16"])
@pytest.mark.parametrize("rows", [1, 63, 64, 65, 8191, 8192, 8193, 100003])
def test_colsum(L, bf16, rows):
    cols_set = (4, 124, 128, 132, 2052) + ((2, 130) if bf16 else (1, 3, 131))   # odd / even tails of the atomic kernel
    dt = BF16 if bf16 else F32
    for cols in cols_set:
        a = _colsum_input(rows, cols, bf16, rows * 7 + cols)
        ref = a.double().sum(0)
        absum = a.double().abs().sum(0)
        ld = cols + (6 if bf16 else 5) if cols % 4 else cols + 12
        buf = _pitched(a, ld)                                         # NaN padding: a read of it poisons the sum
        out = torch.zeros(cols, device="cuda")
        L.check(L.lib().dvt_colsum(_ptr(buf), dt, ld, rows, cols, _ptr(out), _st()), "dvt_colsum")
        assert_within(out.cpu(), ref, _colsum_chain_atomic(rows, cols, bf16, _nsm()) * U * absum, f"colsum {rows}x{cols}")
        if cols % 4:
            continue
        outs = []
        for ld2 in (cols, cols + 8):
            buf2 = _pitched(a, ld2)
            ws = torch.empty(256 * cols, device="cuda")
            for _ in range(2):
                o = torch.full((cols,), math.nan, device="cuda")
                L.check(L.lib().dvt_colsum_ordered(_ptr(buf2), dt, ld2, rows, cols, _ptr(o), _ptr(ws), _st()),
                        "dvt_colsum_ordered")
                outs.append(o.cpu())
        assert_within(outs[0], ref, _chain_ordered(rows) * U * absum, f"colsum_ordered {rows}x{cols}")
        for o in outs[1:]:
            assert torch.equal(o.view(torch.int32), outs[0].view(torch.int32)), "ordered column sum is not reproducible"


# ------------------------------------------------------------------------------------------------ LayerScale / embed backward
@pytest.mark.gpu
@pytest.mark.parametrize("C", [4, 132, 384, 772, 1280])
@pytest.mark.parametrize("rows", [1, 64, 65, 8192, 8193, 20000])
def test_layerscale_bwd(L, C, rows):
    gen = torch.Generator().manual_seed(rows + C)
    dx = torch.randn(rows, C, generator=gen)
    branch = torch.randn(rows, C, generator=gen).bfloat16()
    gamma = (torch.rand(C, generator=gen) + 0.1) * torch.where(torch.rand(C, generator=gen) < 0.5, -1.0, 1.0)
    chain = _chain_ordered(rows)
    for with_gamma in (True, False):
        g = gamma if with_gamma else torch.ones(C)
        dx_buf = _pitched(dx, C + 8)
        dbr = torch.full((rows, C), math.nan, dtype=torch.bfloat16, device="cuda")
        dbias = torch.full((C,), math.nan, device="cuda")
        dgam = torch.full((C,), math.nan, device="cuda") if with_gamma else None
        ws = torch.empty(256 * C, device="cuda")
        br_d, g_d = (branch.cuda(), gamma.cuda()) if with_gamma else (None, None)
        L.check(L.lib().dvt_layerscale_bwd(_ptr(dx_buf), C + 8, _ptr(br_d), _ptr(g_d), _ptr(dbr), _ptr(dbias), _ptr(dgam),
                                           _ptr(ws), rows, C, _st()), "dvt_layerscale_bwd")
        torch.cuda.synchronize()
        prod = g * dx                                                  # fp32 product, as the kernel forms it
        assert torch.equal(dbr.cpu().view(torch.int16), prod.bfloat16().view(torch.int16)), "dbranch != RN-bf16(gamma dx)"
        ref = g.double() * dx.double()
        assert_within(dbias.cpu(), ref.sum(0), (chain + 1) * U * ref.abs().sum(0), f"dbias rows={rows} C={C}")
        if with_gamma:
            t = dx.double() * branch.double()
            assert_within(dgam.cpu(), t.sum(0), chain * U * t.abs().sum(0), f"dgamma rows={rows} C={C}")


@pytest.mark.gpu
@pytest.mark.parametrize("C", [4, 132, 384, 1280])
@pytest.mark.parametrize("B,np_,prefix", [(1, 1, 1), (3, 37, 5), (64, 257, 1), (5, 1369, 5), (2, 8193, 1)])
def test_vit_embed_bwd(L, C, B, np_, prefix):
    ntok = prefix + np_
    gen = torch.Generator().manual_seed(B * np_ + C)
    dx0 = torch.randn(B * ntok, C, generator=gen) + 0.25
    dpatch = torch.full((B * np_, C), math.nan, dtype=torch.bfloat16, device="cuda")
    dpos = torch.full((np_, C), math.nan, device="cuda")
    dpre = torch.full((prefix, C), math.nan, device="cuda")
    dbias = torch.full((C,), math.nan, device="cuda")
    ws = torch.empty(256 * C, device="cuda")
    dx0_d = dx0.cuda()
    L.check(L.lib().dvt_vit_embed_bwd(_ptr(dx0_d), B, ntok, prefix, C, _ptr(dpatch), _ptr(dpos), _ptr(dpre), _ptr(dbias),
                                      _ptr(ws), _st()), "dvt_vit_embed_bwd")
    torch.cuda.synchronize()
    d3 = dx0.view(B, ntok, C)
    assert torch.equal(dpatch.cpu().view(torch.int16), d3[:, prefix:].reshape(B * np_, C).bfloat16().view(torch.int16))
    d64 = d3.double()
    a64 = d64.abs()
    assert_within(dpos.cpu(), d64[:, prefix:].sum(0), B * U * a64[:, prefix:].sum(0), "dpos")
    assert_within(dpre.cpu(), d64[:, :prefix].sum(0), B * U * a64[:, :prefix].sum(0), "dprefix")
    assert_within(dbias.cpu(), d64[:, prefix:].sum((0, 1)), (B + _chain_ordered(np_) + 1) * U * a64[:, prefix:].sum((0, 1)),
                  "dbias")


# ------------------------------------------------------------------------------------------------ token assembly forward
EMBED_NP = (1, 35, 127, 128, 129, 256, 1369)
EMBED_C = (128, 132, 384, 1280)
EMBED_CASES = [(np_, EMBED_C[(i + j) % 4], (1, 3, 5)[(i + j) % 3], (1, 5)[(i + 2 * j) % 2], (i + j) % 2 == 0)
               for i, np_ in enumerate(EMBED_NP) for j in range(4)]


@pytest.mark.gpu
@pytest.mark.parametrize("impl", [0, 1], ids=["tensor_core", "simt"])
def test_vit_embed_fwd(L, impl):
    Kp, K = 592, 588                                                   # 14 x 14 patches: 3 * 196 = 588, padded to 592
    L.check(L.lib().dvt_set_debug_impl(impl))
    try:
        for np_, C, B, prefix, with_bias in EMBED_CASES:
            gen = torch.Generator().manual_seed(np_ * 10 + C + B + prefix)
            patches = torch.zeros(B * np_, Kp, dtype=torch.bfloat16)
            patches[:, :K] = torch.randn(B * np_, K, generator=gen).bfloat16()
            w = torch.zeros(C, Kp, dtype=torch.bfloat16)
            w[:, :K] = (torch.randn(C, K, generator=gen) * 0.05).bfloat16()
            bias = torch.randn(C, generator=gen) if with_bias else None
            pos = torch.randn(np_, C, generator=gen)
            pre = torch.randn(prefix, C, generator=gen)
            ntok = np_ + prefix
            out = torch.full((B * ntok + 130, C), SENT, device="cuda")     # sentinel rows past B * ntok
            out[:B * ntok] = math.nan
            dev = [None if t is None else t.cuda() for t in (patches, w, bias, pos, pre)]   # alive until the kernel ran
            L.check(L.lib().dvt_vit_embed_fwd(_ptr(dev[0]), Kp, _ptr(dev[1]), _ptr(dev[2]), _ptr(dev[3]), _ptr(dev[4]), B, np_,
                                              prefix, C, _ptr(out), _st()), "dvt_vit_embed_fwd")
            torch.cuda.synchronize()
            what = f"embed_fwd np={np_} C={C} B={B} prefix={prefix} bias={with_bias} impl={impl}"
            assert bool((out[B * ntok:] == SENT).all()), f"{what}: store past B * ntok rows"
            o = out[:B * ntok].view(B, ntok, C)
            assert torch.equal(o[:, :prefix].cpu(), pre.expand(B, prefix, C)), f"{what}: prefix rows"
            p64, w64 = patches.cuda().double(), w.cuda().double()
            b64 = torch.zeros(C, dtype=torch.float64, device="cuda") if bias is None else bias.cuda().double()
            ref = (p64 @ w64.T).view(B, np_, C) + b64 + pos.cuda().double()
            P = (p64.abs() @ w64.abs().T).view(B, np_, C) + b64.abs() + pos.cuda().double().abs()
            assert_within(o[:, prefix:], ref, 2.0 ** -18 * P + 2.0 ** -23 * ref.abs(), what)
    finally:
        L.check(L.lib().dvt_set_debug_impl(-1))


# ------------------------------------------------------------------------------------------------ denoising loss
def _loss_inputs(rows, C, seed):
    """Rows cycle through: random; pred = 0; target = 0; pred = 2.5 * target; pred close to target."""
    gen = torch.Generator().manual_seed(seed)
    t = torch.randn(rows, C, generator=gen)
    p = torch.randn(rows, C, generator=gen)
    for r in range(rows):
        k = r % 5
        if k == 1:
            p[r] = 0
        elif k == 2:
            t[r] = 0
        elif k == 3:
            p[r] = 2.5 * t[r]
        elif k == 4:
            p[r] = t[r] + 0.01 * p[r]
    return p, t


@pytest.mark.gpu
@pytest.mark.parametrize("C", C_SET)
def test_denoise_loss(L, C):
    gs = 2.0
    for rows in (1, 7, 8, 9, 4 * _nsm() * 8 + 37):
        p, t = _loss_inputs(rows, C, rows * 3 + C)
        l2_ref, cos_ref, d_ref = loss_ref(p, t, gs)
        bound = loss_dpred_bound(p, t, gs) + 2.0 ** -23 * d_ref.abs()
        blocks = min(4 * _nsm(), (rows + 7) // 8)
        b_l2, b_cos = loss_value_bounds(l2_ref, cos_ref, rows, C, blocks)
        pd, td = p.cuda(), t.cuda()
        dps = []
        for ordered in (False, True):
            dp = torch.full((rows, C), math.nan, device="cuda")
            losses = torch.full((3,), math.nan, device="cuda")
            if ordered:
                ws = torch.empty(2 * ((rows + 7) // 8), device="cuda")
                L.check(L.lib().dvt_denoise_loss_ordered(_ptr(pd), _ptr(td), _ptr(dp), _ptr(losses), _ptr(ws), rows, C, gs,
                                                         _st()), "dvt_denoise_loss_ordered")
            else:
                L.check(L.lib().dvt_denoise_loss(_ptr(pd), _ptr(td), _ptr(dp), _ptr(losses), rows, C, gs, _st()),
                        "dvt_denoise_loss")
            torch.cuda.synchronize()
            what = f"loss rows={rows} C={C} ordered={ordered}"
            lo = losses.cpu().double()
            assert abs(lo[1].item() - l2_ref) <= b_l2, f"{what}: l2 {lo[1].item()} vs {l2_ref}"
            assert abs(lo[2].item() - cos_ref) <= b_cos, f"{what}: cos {lo[2].item()} vs {cos_ref}"
            assert abs(lo[0].item() - (l2_ref + cos_ref)) <= b_l2 + b_cos + U * (l2_ref + cos_ref), what
            assert_within(dp.cpu(), d_ref, bound, f"{what} dpred")
            dps.append(dp.cpu())
        assert torch.equal(dps[0].view(torch.int32), dps[1].view(torch.int32)), "dpred differs between the two kernels"


# ------------------------------------------------------------------------------------------------ AdamW
@pytest.mark.gpu
@pytest.mark.parametrize("wd", [0.0, 0.05])
@pytest.mark.parametrize("big", [False, True], ids=["n4", "grid_stride"])
def test_adamw(L, wd, big):
    n = 2 * 8 * _nsm() * 256 * 4 + 4 if big else 4
    gen = torch.Generator().manual_seed(int(big) * 10 + int(wd * 100))
    p = torch.randn(n, generator=gen)
    grads = torch.randn(n, generator=gen) * 1e-2
    kind = torch.arange(n) % 5
    grads[kind == 1] = 0                                               # exact zeros: the update is exactly the decay
    grads[kind == 2] = torch.randn(int((kind == 2).sum()), generator=gen) * 1e-10   # eps-dominated
    if n == 4:
        grads = torch.tensor([0.0, 3e-3, -1e-10, 0.5])
    zero = grads == 0
    pd, gd = p.cuda(), grads.cuda()
    md, vd = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    for step in (1, 2, 10, 1000, 10 ** 6):
        p0, m0, v0 = pd.cpu(), md.cpu(), vd.cpu()
        L.check(L.lib().dvt_adamw(_ptr(pd), _ptr(gd), _ptr(md), _ptr(vd), n, ADAM["lr"], ADAM["b1"], ADAM["b2"], ADAM["eps"],
                                  wd, step, _st()), "dvt_adamw")
        torch.cuda.synchronize()
        pr, mr, vr, dp, dm, dv = adamw_ref(p0, grads, m0, v0, step, wd)
        what = f"adamw n={n} wd={wd} step={step}"
        assert_within(md.cpu(), mr, dm, f"{what} m")
        assert_within(vd.cpu(), vr, dv, f"{what} v")
        assert_within(pd.cpu(), pr, dp, f"{what} p")
        decay = torch.tensor(1 - ADAM["lr"] * wd, dtype=torch.float32)
        assert torch.equal(pd.cpu()[zero].view(torch.int32), (p0[zero] * decay).view(torch.int32)), f"{what}: zero grad"


# ------------------------------------------------------------------------------------------------ resample backward
def _resample_weights(n_out, n_in, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n_out, n_in, generator=g) * 0.5


@pytest.mark.gpu
@pytest.mark.parametrize("h,w,gh,gw", [(37, 23, 16, 16), (8, 5, 16, 16), (1, 1, 1, 1), (1, 1, 16, 16), (16, 16, 1, 1)])
@pytest.mark.parametrize("C", [1, 3, 384])
def test_resample_bwd(L, h, w, gh, gw, C):
    wh, ww = _resample_weights(h, gh, h + gh), _resample_weights(w, gw, w + gw + 1)
    dout = torch.randn(h, w, C, generator=torch.Generator().manual_seed(C))
    tmp = torch.empty(gh * w * C, device="cuda")
    dgrid = torch.full((gh, gw, C), math.nan, device="cuda")
    dev = [t.cuda() for t in (wh, ww, dout)]                           # alive until the kernel ran
    L.check(L.lib().dvt_resample_bwd(_ptr(dev[0]), _ptr(dev[1]), _ptr(dev[2]), _ptr(tmp), _ptr(dgrid), h, w, gh, gw, C, _st()),
            "dvt_resample_bwd")
    torch.cuda.synchronize()
    ref = torch.einsum("yi,xj,yxc->ijc", wh.double(), ww.double(), dout.double())
    P = torch.einsum("yi,xj,yxc->ijc", wh.double().abs(), ww.double().abs(), dout.double().abs())
    assert_within(dgrid.cpu(), ref, (h + w + 4) * U * P, f"resample_bwd {h}x{w}<-{gh}x{gw} C={C}")


# ------------------------------------------------------------------------------------------------ im2col
@pytest.mark.gpu
@pytest.mark.parametrize("B,H,W,P,S", [(2, 224, 224, 14, 14), (1, 31, 33, 7, 3), (1, 16, 16, 16, 16), (2, 29, 30, 1, 1),
                                       (1, 40, 45, 14, 5), (1, 37, 38, 16, 6), (1, 30, 30, 14, 3), (1, 33, 31, 7, 7)])
@pytest.mark.parametrize("bf16", [False, True], ids=["f32", "bf16"])
@pytest.mark.parametrize("offset", [0, 1], ids=["aligned", "offset1"])
def test_im2col(L, B, H, W, P, S, bf16, offset):
    dt = torch.bfloat16 if bf16 else torch.float32
    x = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(H * W + P)).to(dt)
    flat = torch.empty(x.numel() + 1, dtype=dt, device="cuda")
    flat[offset:offset + x.numel()] = x.reshape(-1).cuda()             # offset 1: a base the paired loads cannot use
    h, w = (H - P) // S + 1, (W - P) // S + 1
    K, Kp = 3 * P * P, (3 * P * P + 7) // 8 * 8
    out = torch.full((B * h * w, Kp), math.nan, dtype=torch.bfloat16, device="cuda")
    L.check(L.lib().dvt_im2col(_ptr(flat, offset), BF16 if bf16 else F32, _ptr(out), B, H, W, P, S, _st()), "dvt_im2col")
    torch.cuda.synchronize()
    ref = F.unfold(x.bfloat16().float(), kernel_size=P, stride=S).transpose(1, 2).reshape(B * h * w, K).bfloat16()
    o = out.cpu()
    assert torch.equal(o[:, :K].view(torch.int16), ref.view(torch.int16)), "im2col != unfold of the bf16 input"
    assert bool((o[:, K:].float() == 0).all()) and not bool(torch.signbit(o[:, K:].float()).any()), "K padding not zero"


# ------------------------------------------------------------------------------------------------ segmentation loss
@pytest.mark.gpu
@pytest.mark.parametrize("K", [2, 33, 64, 65, 96, 97, 161, 255])
@pytest.mark.parametrize("h,w,H,W", [(13, 17, 61, 47), (16, 16, 9, 12)], ids=["up", "down"])
def test_seg_upsample_ce_all_widths(K, h, w, H, W):
    """KV = ceil(K / 32) selects the 1, 2, 3, 5 or 8 register variant.  Labels include K - 1, the values K..254 (no loss
    and no gradient, as the header says) and 255."""
    from dvt.dense_eval import seg_ops
    B = 2
    gen = torch.Generator().manual_seed(K * 100 + H)
    logits = torch.randn(B, h, w, K, generator=gen) * 3
    lab = torch.randint(0, K, (B, H, W), generator=gen)
    r = torch.rand(B, H, W, generator=gen)
    lab[r < 0.1] = K - 1
    if K < 255:
        lab[(r >= 0.1) & (r < 0.2)] = torch.randint(K, 255, (int(((r >= 0.1) & (r < 0.2)).sum()),), generator=gen)
    lab[r > 0.95] = 255
    n = lab.numel()
    ref_in = logits.double().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    up = F.interpolate(ref_in, size=(H, W), mode="bilinear", align_corners=False)
    tgt = torch.where(lab >= K, torch.full_like(lab, 255), lab)
    ref = F.cross_entropy(up, tgt, reduction="sum", ignore_index=255)
    (ref / n).backward()
    ref_grad = ref_in.grad.permute(0, 2, 3, 1)
    loss, dl = seg_ops.upsample_ce_sum(logits.cuda(), lab.to(torch.uint8).cuda(), 1.0 / n)
    assert abs(loss.item() - ref.item()) <= 1e-5 * abs(ref.item()), (loss.item(), ref.item())
    assert (dl.cpu().double() - ref_grad).abs().max() <= 1e-5 * ref_grad.abs().max()
