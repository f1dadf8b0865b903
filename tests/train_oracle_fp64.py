"""fp64 mirror of every autograd node of the stage-2 / stage-3 training step (dvt/train_ops.py), with an error model for
each gradient.  Test infrastructure only.

Teacher forcing.  A node's backward is linear in its incoming gradient once its forward is fixed.  The mirror therefore
takes the node's OWN saved tensors (`y.grad_fn.saved_tensors`, the prepared weights `y.grad_fn.wts`), promotes them to
fp64, and computes every input and parameter gradient from them in fp64.  It follows the math of the node (timm Block /
oracle/vit.py `block`, the oracle/denoiser.py block, the loss of main_denoiser.py:214-217, separable bicubic resampling),
not the code of train_ops.py: attention probabilities are read as the kernel forms them, P = exp2(s log2e - lse_saved),
and delta = rowsum(dout * out) is formed from the saved bf16 `out`.

Error model.  Every gradient is carried as a pair G(val, var): the fp64 value and the variance of the error a rounding
implementation accumulates on the way.  The variance pass is the same backward on squared magnitudes with every fixed
factor squared (the map from the incoming gradient to every output is linear, so an error e entering at one stage reaches
an output as L e, and independent errors add their variances).  Stages that inject error:
  * each bf16 rounding of the backward -- d2, dhpre, d1, datt, dqkv, the second rounding by dvt_rope_bwd, and inside the
    attention backward P (for dV) and dS -- injects (U_B |value|)^2.  U_B = 2^-9 is the rms relative error of
    round-to-nearest bf16 (an ulp of 2^-8 .. 2^-7 relative, uniform error of ulp / sqrt(12)), not its worst case 2^-8;
  * an fp32 sum of depth D (GEMM accumulation, column sums, LayerNorm row sums) injects D (U_32 sum|terms|)^2, the
    variance form of the probabilistic bound of Higham & Mary (SIAM J. Sci. Comput. 41(5), 2019);
  * the epilogue approximations of test_gemm_conformance_gpu.py: the fast-erf GELU derivative, 2e-6 |acc| absolute, and
    the SiLU factors of the SwiGLU backward, 2^-20 |value|.
The check is |g - g64| <= LAMBDA sqrt(var) per element.  No branch ambiguity arises (GELU, SiLU, softmax, LayerNorm and
the cosine loss are smooth), so there is no allowance term.  Caveat: errors of correlated paths are treated as
independent.  In dS = P (dP - delta), dP and delta see the same dout error, and their covariance is dropped; this can
understate the variance by up to 2x.  LAMBDA covers it.  One correlation is structural and handled explicitly: a dout
error reaches every dV_j through P, whose rows sum to 1, so sums over the rows of dV add it coherently (see `attn_bwd`).
LAMBDA = 10 was fixed from the honest bf16 emulation of test_train_oracle_fp64_cpu.py: over every block option and three
seeds the worst |g - g64| / sqrt(var) there is 4.0 (the rms is ~1), so the check leaves 2.5x of room.

Forward conformance.  `check_*_forward` and `ln_excess` compare each saved activation with fp64 of its op applied to the preceding SAVED
activation, with the per-op bounds of test_gemm_conformance_gpu.py, test_attention_conformance_gpu.py and
test_train_kernels_conformance_gpu.py (restated here, not imported)."""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Optional

import torch
import torch.nn.functional as F

U_B = 2.0 ** -9
U_32 = 2.0 ** -24
LAMBDA = 10.0
GELU_GRAD_ABS = 2e-6         # fast-erf GELU derivative of the dgrad epilogue, times |acc|
SILU_REL = 2.0 ** -20        # __expf and the fp32 sigmoid of the SwiGLU backward epilogue, relative
LOG2E = 1.0 / math.log(2.0)


# ------------------------------------------------------------------------------------------------ gradient + variance
@dataclass
class G:
    val: torch.Tensor
    var: torch.Tensor

    def __add__(self, o: "G") -> "G":
        return G(self.val + o.val, self.var + o.var)

    def mul(self, f) -> "G":
        """Times a fixed factor (broadcast)."""
        return G(self.val * f, self.var * (f * f))

    def __getitem__(self, idx) -> "G":
        return G(self.val[idx], self.var[idx])

    def reshape(self, *s) -> "G":
        return G(self.val.reshape(*s), self.var.reshape(*s))


def exact(t: torch.Tensor) -> G:
    t = t.detach().double()
    return G(t, torch.zeros_like(t))


def rnd(g: G) -> G:
    """A bf16 rounding of the value."""
    return G(g.val, g.var + (U_B * g.val) ** 2)


def _acc(var: torch.Tensor, depth: int, absum: torch.Tensor) -> torch.Tensor:
    return var + depth * (U_32 * absum) ** 2


def mm(g: G, w: torch.Tensor) -> G:
    """g [M, K] @ w [K, N], fp32 accumulation."""
    return G(g.val @ w, _acc(g.var @ (w * w), w.shape[0], g.val.abs() @ w.abs()))


def wgrad(dy: G, x: torch.Tensor) -> G:
    """dy^T x: dW [out, in] of a linear layer over the rows."""
    return G(dy.val.t() @ x, _acc(dy.var.t() @ (x * x), x.shape[0], dy.val.abs().t() @ x.abs()))


def colsum(g: G) -> G:
    return G(g.val.sum(0), _acc(g.var.sum(0), g.val.shape[0], g.val.abs().sum(0)))


def rowdot(g: G, f: torch.Tensor) -> G:
    """sum_rows g * f (a LayerScale dgamma)."""
    return colsum(g.mul(f))


def ln_bwd(x: torch.Tensor, gamma: torch.Tensor, dy: G, eps: float):
    """LayerNorm backward at the fp32 input x (f64 here): (dx, dgamma, dbeta)."""
    C = x.shape[1]
    mu = x.mean(1, keepdim=True)
    rstd = ((x - mu).pow(2).mean(1, keepdim=True) + eps).rsqrt()
    xh = (x - mu) * rstd
    gd = dy.mul(gamma)
    m1, m2 = gd.val.mean(1, keepdim=True), (gd.val * xh).mean(1, keepdim=True)
    dx = rstd * (gd.val - m1 - xh * m2)
    v1, v2 = gd.var.sum(1, keepdim=True) / C ** 2, (gd.var * xh * xh).sum(1, keepdim=True) / C ** 2
    dx_var = rstd ** 2 * (gd.var + v1 + xh * xh * v2)
    mag = rstd * (gd.val.abs() + gd.val.abs().mean(1, keepdim=True) + xh.abs() * (gd.val * xh).abs().mean(1, keepdim=True))
    dx_var = _acc(dx_var, C, mag)
    return G(dx, dx_var), rowdot(dy, xh), colsum(dy)


def gelu_grad(x: torch.Tensor) -> torch.Tensor:
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def rope_rot(t: torch.Tensor, cos: torch.Tensor, sin: torch.Tensor, sign: float) -> torch.Tensor:
    """Rotate the (d, d + 32) pairs of t [..., rows, heads, 64] by +angle (sign 1, the forward) or -angle (sign -1)."""
    lo, hi = t[..., :32], t[..., 32:]
    c, s = cos[:, None, :], sign * sin[:, None, :]
    return torch.cat([lo * c - hi * s, hi * c + lo * s], -1)


def rope_bwd(dqkv: G, table: torch.Tensor, batch: int, prefix: int, heads: int) -> G:
    """Transpose of the RoPE rotation on the q / k columns of the patch rows, then a bf16 rounding (dvt_rope_bwd)."""
    M, C3 = dqkv.val.shape
    C = C3 // 3
    ntok = M // batch
    cos, sin = table[:, :32].double(), table[:, 32:].double()
    val = dqkv.val.clone().view(batch, ntok, 3, heads, C // heads)
    var = dqkv.var.clone().view(batch, ntok, 3, heads, C // heads)
    for j in range(2):
        pv, pq = val[:, prefix:, j], var[:, prefix:, j]
        val[:, prefix:, j] = rope_rot(pv, cos, sin, -1.0)
        var[:, prefix:, j] = torch.cat([pq[..., :32] * cos[:, None] ** 2 + pq[..., 32:] * sin[:, None] ** 2,
                                        pq[..., 32:] * cos[:, None] ** 2 + pq[..., :32] * sin[:, None] ** 2], -1)
        # the second bf16 rounding, on the rotated rows only
        var[:, prefix:, j] += (U_B * val[:, prefix:, j]) ** 2
    return G(val.view(M, C3), var.view(M, C3))


def attn_probs(qkv: torch.Tensor, lse: torch.Tensor, batch: int, heads: int):
    """(q, k, v [B, H, N, D] f64, P [B, H, N, N] = exp2(s log2e - lse), scale) from the saved qkv and lse."""
    M, C3 = qkv.shape
    N, D = M // batch, C3 // 3 // heads
    t = qkv.double().view(batch, N, 3, heads, D).permute(2, 0, 3, 1, 4)
    q, k, v = t[0], t[1], t[2]
    scale = D ** -0.5
    s = (q @ k.transpose(-1, -2)) * scale
    P = torch.exp2(s * LOG2E - lse.double()[..., None])
    return q, k, v, P, scale


def attn_bwd(qkv: torch.Tensor, out: torch.Tensor, dout: G, lse: torch.Tensor, batch: int, heads: int) -> G:
    """Flash-attention backward in fp64 from the saved qkv / out / lse; dqkv before its bf16 rounding."""
    M, C3 = qkv.shape
    C = C3 // 3
    N, D = M // batch, C // heads
    q, k, v, P, scale = attn_probs(qkv, lse, batch, heads)
    hv = lambda t: t.view(batch, N, heads, D).permute(0, 2, 1, 3)          # noqa: E731
    dO, vO, O = hv(dout.val), hv(dout.var), hv(out.double())
    dV = P.transpose(-1, -2) @ dO
    # dout's error e_i reaches every dV_j with the weight P_ij, and sum_j P_ij = 1: later sums over the rows j (the v-bias
    # and the QKV weight gradient) add those shares coherently.  Carrying P instead of P^2 bounds every such sum by
    # Cauchy-Schwarz, (sum_j P_ij a_j)^2 <= sum_j P_ij a_j^2.
    dV_var = P.transpose(-1, -2) @ vO + (U_B ** 2) * (P * P).transpose(-1, -2) @ (dO * dO)   # bf16 P
    dV_var = _acc(dV_var, N, P.transpose(-1, -2) @ dO.abs())
    dP = dO @ v.transpose(-1, -2)
    dP_var = _acc(vO @ (v * v).transpose(-1, -2), D, dO.abs() @ v.abs().transpose(-1, -2))
    delta = (dO * O).sum(-1, keepdim=True)
    delta_var = _acc((vO * O * O).sum(-1, keepdim=True), D, (dO * O).abs().sum(-1, keepdim=True))
    dS = P * (dP - delta) * scale
    dS_var = (P * scale) ** 2 * (dP_var + delta_var) + (U_B * dS) ** 2                             # bf16 dS
    dQ = dS @ k
    dQ_var = _acc(dS_var @ (k * k), N, dS.abs() @ k.abs())
    dK = dS.transpose(-1, -2) @ q
    dK_var = _acc(dS_var.transpose(-1, -2) @ (q * q), N, dS.abs().transpose(-1, -2) @ q.abs())
    back = lambda t: t.permute(0, 2, 1, 3).reshape(M, C)                   # noqa: E731
    return G(torch.cat([back(dQ), back(dK), back(dV)], 1), torch.cat([back(dQ_var), back(dK_var), back(dV_var)], 1))


# ------------------------------------------------------------------------------------------------ nodes
BLOCK_WTS = ("n1w", "n1b", "wq", "qkvb", "wp", "projb", "ls1", "n2w", "n2b", "w1", "fc1b", "w2", "fc2b", "ls2")
BLOCK_ACTS = ("x1", "xn1", "qkv", "att", "lse", "br1", "xn2", "hpre", "hid", "br2")


def _d(t):
    return None if t is None else t.detach().double()


def block_bwd(x0, acts: Dict[str, torch.Tensor], wts: Dict[str, Optional[torch.Tensor]], dx2: G, *, heads: int, batch: int,
              eps: float, rope=None) -> Dict[str, G]:
    """Backward of one pre-LN block (`_VitBlockFn`; `_BlockFn` is the case without LayerScale, eps 1e-6, GELU) from the
    saved activations.  Returns the gradients under the names of `BLOCK_WTS` (w* -> the weight) and "x0"."""
    a = {k: _d(v) for k, v in acts.items()}
    w = {k: _d(v) for k, v in wts.items()}
    x0 = _d(x0)
    M, C = x0.shape
    swiglu = 2 * w["w2"].shape[1] == w["w1"].shape[0]
    out: Dict[str, G] = {}
    # ---- MLP branch ----
    d2 = dx2 if w["ls2"] is None else dx2.mul(w["ls2"])
    out["fc2b"] = colsum(d2)
    if w["ls2"] is not None:
        out["ls2"] = rowdot(dx2, a["br2"])
    d2 = rnd(d2)
    out["w2"] = wgrad(d2, a["hid"])
    dh = mm(d2, w["w2"])
    if swiglu:
        Hh = w["w2"].shape[1]
        g, u = a["hpre"][:, :Hh], a["hpre"][:, Hh:]
        s = torch.sigmoid(g)
        fg, fu = u * (s + g * s * (1 - s)), g * s
        dhpre = G(torch.cat([dh.val * fg, dh.val * fu], 1), torch.cat([dh.var * fg * fg, dh.var * fu * fu], 1))
        dhpre.var = dhpre.var + (SILU_REL * dhpre.val) ** 2
    else:
        gp = gelu_grad(a["hpre"])
        dhpre = dh.mul(gp)
        dhpre.var = dhpre.var + (GELU_GRAD_ABS * dh.val) ** 2
    dhpre = rnd(dhpre)
    out["w1"] = wgrad(dhpre, a["xn2"])
    out["fc1b"] = colsum(dhpre)
    dxn2 = mm(dhpre, w["w1"])
    dln, out["n2w"], out["n2b"] = ln_bwd(a["x1"], w["n2w"], dxn2, eps)
    dx1 = dx2 + dln
    dx1.var = dx1.var + (U_32 * dx1.val) ** 2
    # ---- attention branch ----
    d1 = dx1 if w["ls1"] is None else dx1.mul(w["ls1"])
    out["projb"] = colsum(d1)
    if w["ls1"] is not None:
        out["ls1"] = rowdot(dx1, a["br1"])
    d1 = rnd(d1)
    out["wp"] = wgrad(d1, a["att"])
    datt = rnd(mm(d1, w["wp"]))
    dqkv = rnd(attn_bwd(a["qkv"], a["att"], datt, acts["lse"], batch, heads))
    if rope is not None:
        dqkv = rope_bwd(dqkv, rope[0], batch, rope[1], heads)
    out["wq"] = wgrad(dqkv, a["xn1"])
    out["qkvb"] = colsum(dqkv)
    if rope is not None:      # no key bias: its gradient is defined as zero
        out["qkvb"].val[C:2 * C] = 0
        out["qkvb"].var[C:2 * C] = 0
    dxn1 = mm(dqkv, w["wq"])
    dln, out["n1w"], out["n1b"] = ln_bwd(x0, w["n1w"], dxn1, eps)
    out["x0"] = dx1 + dln
    out["x0"].var = out["x0"].var + (U_32 * out["x0"].val) ** 2
    return out


def embed_bwd(patches: torch.Tensor, dx0: G, *, batch: int, prefix: int, C: int, P: int) -> Dict[str, G]:
    """`_VitEmbedFn` backward: pe_w [C, 3, P, P], pe_b, pos_patch [np, C], prefix_rows [prefix, C]."""
    ntok = dx0.val.shape[0] // batch
    t = dx0.reshape(batch, ntok, C)
    pat = t[:, prefix:]
    pre = t[:, :prefix]
    sum0 = lambda g: G(g.val.sum(0), _acc(g.var.sum(0), g.val.shape[0], g.val.abs().sum(0)))   # noqa: E731
    K = 3 * P * P
    dpatch = rnd(pat.reshape(-1, C))
    gw = wgrad(dpatch, patches.double()[:, :K])
    return {"pe_w": gw.reshape(C, 3, P, P), "pe_b": colsum(pat.reshape(-1, C)), "pos": sum0(pat), "prefix": sum0(pre)}


def layernorm_bwd(x: torch.Tensor, w: torch.Tensor, dy: G, eps: float) -> Dict[str, G]:
    """`_VitLayerNormFn` backward (norm_pre)."""
    dx, dg, db = ln_bwd(x.double(), w.double(), dy, eps)
    return {"x": dx, "w": dg, "b": db}


def norm_strip_bwd(x: torch.Tensor, w: torch.Tensor, dy: G, *, ntok: int, prefix: int, eps: float) -> Dict[str, G]:
    """`_VitNormStripFn` backward: LayerNorm over the patch rows of every image, the prefix rows get exactly zero."""
    M, C = x.shape
    B = M // ntok
    xk = x.double().view(B, ntok, C)[:, prefix:].reshape(-1, C)
    dxk, dg, db = ln_bwd(xk, w.double(), dy, eps)
    val = torch.zeros(B, ntok, C, dtype=torch.float64, device=x.device)
    var = torch.zeros_like(val)
    val[:, prefix:] = dxk.val.view(B, -1, C)
    var[:, prefix:] = dxk.var.view(B, -1, C)
    return {"x": G(val.view(M, C), var.view(M, C)), "w": dg, "b": db}


def loss_bwd(pred: torch.Tensor, target: torch.Tensor, g_total: float = 1.0) -> G:
    """d(l2 + 1 - mean cos)/d pred (main_denoiser.py:214-217) in fp64, with the fp32 error of dvt_denoise_loss."""
    C = pred.shape[-1]
    p = pred.detach().double().reshape(-1, C)
    t = target.detach().double().reshape(-1, C)
    n = p.shape[0]
    pn = p.norm(dim=1, keepdim=True).clamp_min(1e-8)
    tn = t.norm(dim=1, keepdim=True).clamp_min(1e-8)
    cos = (p * t).sum(1, keepdim=True) / (pn * tn)
    val = g_total * (2.0 * (p - t) / (n * C) - (t / (pn * tn) - cos * p / pn ** 2) / n)
    mag = abs(g_total) * (2.0 * (p - t).abs() / (n * C) + (t.abs() / (pn * tn) + p.abs() / pn ** 2) / n)
    return G(val, C * (U_32 * mag) ** 2 + (U_32 * val) ** 2)


def resample_weights64(n_in: int, n_out: int, device) -> torch.Tensor:
    """f64 [n_out, n_in] weights of bicubic antialiased interpolation along one axis (the separable 1-D operator)."""
    eye = torch.eye(n_in, dtype=torch.float64).reshape(1, n_in, 1, n_in)
    return F.interpolate(eye, size=(1, n_out), mode="bicubic", antialias=True)[0, :, 0, :].t().contiguous().to(device)


def resample_bwd(dout: G, gh: int, gw: int) -> G:
    """`_ResampleFn` backward: dout [1, C, h, w] -> d grid [1, C, gh, gw] = Wh^T dout Ww."""
    _, C, h, w = dout.val.shape
    dev = dout.val.device
    wh, ww = resample_weights64(gh, h, dev), resample_weights64(gw, w, dev)
    v = torch.einsum("ai,cab,bj->cij", wh, dout.val[0], ww)
    var = torch.einsum("ai,cab,bj->cij", wh * wh, dout.var[0], ww * ww)
    mag = torch.einsum("ai,cab,bj->cij", wh.abs(), dout.val[0].abs(), ww.abs())
    # + the fp32 weights themselves: ATen evaluates the cubic filter and normalises it in fp32, a few ulps per weight
    return G(v[None], _acc(var, h + w, mag)[None] + (8 * U_32 * mag[None]) ** 2)


# ------------------------------------------------------------------------------------------------ fp64 forward
def ln64(x, w, b, eps):
    return F.layer_norm(x.double(), (x.shape[1],), _d(w), _d(b), eps)


def block_fwd64(x0, wts, *, heads: int, batch: int, eps: float, rope=None, round_to=None):
    """The block forward in fp64 producing the activations `_vit_block_fwd` keeps (for the host-side checks): round_to
    None keeps fp64, "bf16" rounds the saved tensors as the kernels store them (bf16 GEMM operands, fp32 residual
    stream).  Returns (x2, acts)."""
    w = {k: _d(v) for k, v in wts.items()}
    b16 = (lambda t: t.bfloat16().double()) if round_to == "bf16" else (lambda t: t)     # noqa: E731
    f32 = (lambda t: t.float().double()) if round_to == "bf16" else (lambda t: t)        # noqa: E731
    x0 = _d(x0)
    M, C = x0.shape
    N, D = M // batch, C // heads
    xn1 = b16(ln64(x0, w["n1w"], w["n1b"], eps))
    qkv = xn1 @ w["wq"].t() + w["qkvb"]
    if rope is not None:
        qkv = qkv_rope(qkv, rope[0].double(), batch, rope[1], heads)
    qkv = b16(qkv)
    t = qkv.view(batch, N, 3, heads, D).permute(2, 0, 3, 1, 4)
    s = (t[0] @ t[1].transpose(-1, -2)) * D ** -0.5
    lse = f32(torch.logsumexp(s, -1) * LOG2E)
    att = b16((torch.softmax(s, -1) @ t[2]).permute(0, 2, 1, 3).reshape(M, C))
    br1 = att @ w["wp"].t() + w["projb"]
    x1 = f32(x0 + (br1 if w["ls1"] is None else br1 * w["ls1"]))
    xn2 = b16(ln64(x1, w["n2w"], w["n2b"], eps))
    hpre = b16(xn2 @ w["w1"].t() + w["fc1b"])
    if 2 * w["w2"].shape[1] == w["w1"].shape[0]:
        Hh = w["w2"].shape[1]
        hid = b16(F.silu(hpre[:, :Hh]) * hpre[:, Hh:])
    else:
        hid = b16(F.gelu(hpre))
    br2 = hid @ w["w2"].t() + w["fc2b"]
    x2 = f32(x1 + (br2 if w["ls2"] is None else br2 * w["ls2"]))
    acts = dict(x1=x1, xn1=xn1, qkv=qkv, att=att, lse=lse, br1=None if w["ls1"] is None else b16(br1), xn2=xn2, hpre=hpre,
                hid=hid, br2=None if w["ls2"] is None else b16(br2))
    return x2, acts


def qkv_rope(qkv: torch.Tensor, table: torch.Tensor, batch: int, prefix: int, heads: int) -> torch.Tensor:
    """The RoPE of the QKV epilogue: q and k of the patch rows rotated (bias included)."""
    M, C3 = qkv.shape
    C = C3 // 3
    t = qkv.clone().view(batch, M // batch, 3, heads, C // heads)
    for j in range(2):
        t[:, prefix:, j] = rope_rot(t[:, prefix:, j], table[:, :32], table[:, 32:], 1.0)
    return t.view(M, C3)


# ------------------------------------------------------------------------------------------------ checks
def ratio(got: torch.Tensor, ref: G, lam: float = LAMBDA):
    """(worst |got - ref| / (lam sqrt(var)), rms of the ratio at lam = 1); NaN counts as infinitely far."""
    err = (got.detach().double().to(ref.val.device) - ref.val).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    sd = ref.var.sqrt() + 1e-300
    r = err / sd
    return (r.max().item() / lam if r.numel() else 0.0), (r.pow(2).mean().sqrt().item() if r.numel() else 0.0)


def forward_excess(got, ref, P, *, rel=2.0 ** -17, bf16_out=False):
    """Forward conformance of one saved tensor: |got - ref| <= rel P + 2^-23 |ref| (+ 2^-8 |ref| for a bf16 store),
    P the op's absolute envelope.  Returns the worst ratio to the bound."""
    ref = ref.double()
    bound = rel * P + 2.0 ** -23 * ref.abs() + 1e-30
    if bf16_out:
        bound = bound + 2.0 ** -8 * ref.abs()
    err = (got.detach().double() - ref).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    return (err / bound).max().item()


def ln_excess(got, x, w, b, eps, *, bf16_out=False):
    """LayerNorm forward conformance (test_train_kernels_conformance_gpu.py): with sigma_e = sqrt(var + eps),
    m = max|x| of the row and xhat = (x - mean) / sigma_e,
      |y - ref| <= 2^-17 |gamma| (1 + |xhat|)(1 + m / sigma_e) + 2^-23 (|ref| + |beta|);
    a bf16 store adds its rounding, 2^-8 |y| <= 2^-8 |ref| + 2^-8 of the fp32 bound.  Returns the worst ratio."""
    x = x.double()
    w, b = w.double(), b.double()
    ref = ln64(x, w, b, eps)
    mu = x.mean(1, keepdim=True)
    sig = ((x - mu).pow(2).mean(1, keepdim=True) + eps).sqrt()
    xh = (x - mu) / sig
    m = x.abs().amax(1, keepdim=True)
    bound = 2.0 ** -17 * w.abs() * (1 + xh.abs()) * (1 + m / sig) + 2.0 ** -23 * (ref.abs() + b.abs())
    if bf16_out:
        bound = (1 + 2.0 ** -8) * bound + 2.0 ** -8 * ref.abs()
    err = (got.detach().double() - ref).abs()
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    return (err / (bound + 1e-300)).max().item()


def check_embed_forward(out, patches, pe_w, pe_b, pos_patch, prefix_rows, *, batch: int) -> Dict[str, float]:
    """`_VitEmbedFn` output against fp64 of the patch GEMM on the saved bf16 patches and the bf16 weights it multiplies,
    + bias + pos (|out - ref| <= 2^-18 P + 2^-23 |ref|, P = |patches| |W|^T + |bias| + |pos|); the prefix rows must equal
    prefix_rows exactly."""
    C = pe_w.shape[0]
    K = pe_w[0].numel()
    wb = pe_w.detach().float().reshape(C, K).bfloat16().double()
    pa = patches.double()[:, :K]
    ref, P = pa @ wb.t(), pa.abs() @ wb.abs().t()
    for t in (pe_b, pos_patch):
        if t is not None:
            t = t.detach().double()
            ref = (ref.view(batch, -1, C) + t).view(-1, C)
            P = (P.view(batch, -1, C) + t.abs()).view(-1, C)
    prefix = prefix_rows.shape[0]
    o = out.detach().view(batch, -1, C)
    exact_prefix = torch.equal(o[:, :prefix], prefix_rows.detach().float().expand(batch, -1, -1))
    r = forward_excess(o[:, prefix:].reshape(-1, C), ref, P, rel=2.0 ** -18)
    return {"patch rows": r, "prefix rows": 0.0 if exact_prefix else math.inf}


def check_block_forward(x0, acts, wts, x2, *, heads: int, batch: int, eps: float, rope=None) -> Dict[str, float]:
    """Each saved activation of a block against fp64 of its op on the preceding saved activation: worst ratio per tensor."""
    w = {k: _d(v) for k, v in wts.items()}
    a = {k: _d(v) for k, v in acts.items()}
    x0 = _d(x0)
    M, C = x0.shape
    N, D = M // batch, C // heads
    r = {}
    r["xn1"] = ln_excess(a["xn1"], x0, w["n1w"], w["n1b"], eps, bf16_out=True)
    pre = a["xn1"] @ w["wq"].t() + w["qkvb"]
    Pq = a["xn1"].abs() @ w["wq"].abs().t() + w["qkvb"].abs()
    if rope is not None:
        tb = rope[0].double()
        pre = qkv_rope(pre, tb, batch, rope[1], heads)
        Pq = qkv_rope(Pq, tb.abs(), batch, rope[1], heads).abs() + Pq   # |cos| P + |sin| P' (loose by at most 2x)
    r["qkv"] = forward_excess(a["qkv"], pre, Pq, rel=2.0 ** -18 * 4, bf16_out=True)
    q, k, v, Pm, _ = attn_probs(acts["qkv"], acts["lse"], batch, heads)
    s = (q @ k.transpose(-1, -2)) * D ** -0.5
    ref_o = (torch.softmax(s, -1) @ v)
    got_o = a["att"].view(batch, N, heads, D).permute(0, 2, 1, 3)
    vmax = v.abs().amax(dim=(2, 3), keepdim=True)
    r["att"] = ((got_o - ref_o).abs() / (2.0 ** -7 * vmax + 2.0 ** -8 * ref_o.abs())).max().item()
    r["lse"] = (a["lse"] - torch.logsumexp(s, -1) * LOG2E).abs().max().item() / 2e-3
    br1 = a["att"] @ w["wp"].t() + w["projb"]
    Pb1 = a["att"].abs() @ w["wp"].abs().t() + w["projb"].abs()
    ls1 = 1.0 if w["ls1"] is None else w["ls1"]
    r["x1"] = forward_excess(a["x1"], x0 + br1 * ls1, 2.0 * Pb1 * (ls1 if w["ls1"] is None else ls1.abs()) + x0.abs() / 2)
    if a.get("br1") is not None:
        r["br1"] = forward_excess(a["br1"], br1, 2.0 * Pb1, bf16_out=True)
    r["xn2"] = ln_excess(a["xn2"], a["x1"], w["n2w"], w["n2b"], eps, bf16_out=True)
    hp = a["xn2"] @ w["w1"].t() + w["fc1b"]
    r["hpre"] = forward_excess(a["hpre"], hp, 4.0 * (a["xn2"].abs() @ w["w1"].abs().t() + w["fc1b"].abs()), bf16_out=True)
    if 2 * w["w2"].shape[1] == w["w1"].shape[0]:
        Hh = w["w2"].shape[1]
        g, u = a["hpre"][:, :Hh], a["hpre"][:, Hh:]
        r["hid"] = forward_excess(a["hid"], F.silu(g) * u, 8.0 * (F.silu(g) * u).abs(), bf16_out=True)
    else:
        r["hid"] = forward_excess(a["hid"], F.gelu(a["hpre"]), torch.full_like(a["hpre"], 1e-6 / 2.0 ** -17), bf16_out=True)
    br2 = a["hid"] @ w["w2"].t() + w["fc2b"]
    Pb2 = a["hid"].abs() @ w["w2"].abs().t() + w["fc2b"].abs()
    ls2 = 1.0 if w["ls2"] is None else w["ls2"]
    r["x2"] = forward_excess(x2, a["x1"] + br2 * ls2, 2.0 * Pb2 * (ls2 if w["ls2"] is None else ls2.abs()) + a["x1"].abs() / 2)
    if a.get("br2") is not None:
        r["br2"] = forward_excess(a["br2"], br2, 2.0 * Pb2, bf16_out=True)
    return r
