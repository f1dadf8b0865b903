"""fp64 oracle of ONE step of the stage-1 fit, with a rounding-error envelope for every gradient.  Test infrastructure only.

Built on oracle/fit.py and oracle/hashgrid.py, which it reuses unchanged.  Given the fp32 optimiser state S_t (p, m, v of
the twelve tensors of oracle/fit.py::PARAM_ORDER, in the reference layouts), the bank rows of step t and the schedule
scalars, `step` returns the five loss terms, the gradient g of every tensor (loss_scale applied, never unscaled, as the
reference does) and what the engine's state S_{t+1} has to be.

Discrete decisions stay in fp32, exactly as the reference makes them: the hash-grid corners and weights come from
`HG.corner_indices_weights` on the fp32 coordinates, and the grid_sample node weights of G from
`dvt.fit.artifact_axis_table` (with the ~1e-6 share that 9 of 37 nodes leak into a neighbouring cell).  Everything after
them is fp64.  The forward is the full grid_sample (all four corners), not the engine's main-cell shortcut.

Error model.  Alongside each gradient g the oracle evaluates the envelope E: the same forward and backward on the
absolute value of every factor and every summand (|dY|^T |[X | 1]| for a weight gradient, sum_k w_k |d enc| for a table
entry, ...).  An fp32 evaluation of a sum of products in any order and with any blocking satisfies
|g32 - g| <= c * 2^-24 * E, where c grows with the number of roundings on the way.  The engine's c is stated per stage:

  * 3xTF32 product (hi*hi + hi*lo + lo*hi, lo*lo dropped, lo read by the tensor core with a 10-bit mantissa):
    <= 2^-21 + 2^-21 + 2^-22 = 20 * 2^-24 relative per product; with the roundings of the hi / lo split, 24.
  * accumulation of depth D in fp32 (D = 3 K / 8 for wgmma: one fp32 addition per k-group of 8 and product pass;
    D = 3 K for the SIMT debug GEMMs: one fma per product and pass): the probabilistic bound of Higham & Mary
    (SIAM J. Sci. Comput. 41(5), 2019), lambda * sqrt(D) * u with lambda = 8 (failure probability per element
    < 2 exp(-32) ~ 3e-14, negligible over the ~1e9 elements a full run checks) -- a worst-case D * u would be so loose that
    a GEMM computed at TF32 accuracy (2^-11 relative per product) would pass.  The reductions of the loss kernel
    (per-lane sums of C / 32 elements and five shuffle levels) and the ordered sums of the table / G scatter use the same
    rule with their own depths.
  * stages compose: the error a stage inherits through its inputs is bounded by the envelope of the inputs times the
    stage's absolute values, so the c of a gradient is the quadrature sum of the c of every stage on its longest
    dependency path (independent rounding errors of different stages add in quadrature under the same model).

Ambiguity allowance A.  A ReLU pre-activation z, or a residual output q (the sign(q) of the sparsity term), whose
magnitude is below a running bound of its fp32 error (each stage's c u |x| |W|^T on the actual |inputs|, plus the inputs'
bounds carried through W in quadrature: tighter than c u E, which compounds the looseness of every layer) is within rounding of its
decision point, so the fp32 engine may take the other branch.
For every such element the oracle adds the magnitude of the other branch's contribution to A of every gradient it
reaches; the checks are |g32 - g| <= c u E + A.  `n_ambiguous` counts these elements, and the GPU tests require the
gradient elements that pass only through A to stay under 1 % of a tensor, so an unusual seed where the allowance would
carry a tensor fails instead of passing silently.

Adam.  torch.optim.Adam as the reference drives it (oracle/fit.py): L2 decay folded into the gradient, betas (0.9, 0.99),
eps 1e-15 added outside the square root, per-tensor step counters; the per-step scalars lr / (1 - 0.9^t) and
1 / sqrt(1 - 0.99^t) are computed in double and rounded to float, as the engine's host code does.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict

import numpy as np
import torch

from oracle import fit as OF
from oracle import hashgrid as HG

U = 2.0 ** -24
LAMBDA = 8.0
C_PRODUCT = 24.0
RESIDUAL = ["res.0.weight", "res.0.bias", "res.2.weight", "res.2.bias", "res.4.weight", "res.4.bias"]


def c_gemm(K: int, simt: bool = False) -> float:
    """c of one 3xTF32 GEMM with reduction length K (see the module docstring)."""
    depth = 3 * K if simt else 3 * math.ceil(K / 8)
    return C_PRODUCT + LAMBDA * math.sqrt(depth)


def c_sum(depth: int) -> float:
    """c of an fp32 sum of `depth` terms (plus the rounding of each product term)."""
    return 2.0 + LAMBDA * math.sqrt(max(depth, 1))


def quad(*cs: float) -> float:
    return math.sqrt(sum(c * c for c in cs))


def axis_tables(size: int, exact: bool):
    """Per node of one axis: first cell, weight of that cell, weight of the next one (fp32 values promoted to fp64)."""
    if exact:
        from dvt.fit import artifact_axis_table
        i0, w0, w1 = artifact_axis_table(size)
        return i0.long(), w0.double(), w1.double()
    i = torch.arange(size)
    return i, torch.ones(size, dtype=torch.float64), torch.zeros(size, dtype=torch.float64)


@dataclass
class Scalars:
    lr: float          # learning rate of this step (oracle/fit.py::lr_at)
    t: int             # Adam step counter of the main tensors (1 at step 0)
    tr: int            # Adam step counter of the residual MLP (0: not trained at this step)
    phase2: bool
    wd: float
    loss_scale: float

    def adam(self, residual: bool):
        t = self.tr if residual else self.t
        ss = np.float32(self.lr / (1.0 - 0.9 ** t))
        ibc = np.float32(1.0 / math.sqrt(1.0 - 0.99 ** t))
        return float(ss), float(ibc)


def scalars_at(step: int, *, lr, min_lr, warmup_iters, num_iters, freeze_after, weight_decay, loss_scale) -> Scalars:
    freeze_step = int(freeze_after * num_iters)
    phase2 = step > freeze_step
    return Scalars(OF.lr_at(step, lr, min_lr, warmup_iters, num_iters), step + 1, step - freeze_step if phase2 else 0,
                   phase2, weight_decay, loss_scale)


@dataclass
class StepResult:
    losses: Dict[str, float]
    loss_tol: Dict[str, float]          # bound of |fp32 loss - fp64 loss|
    grad: Dict[str, torch.Tensor]       # fp64, reference layouts, loss_scale applied, weight decay NOT included
    env: Dict[str, torch.Tensor]        # envelope E of each gradient
    allow: Dict[str, torch.Tensor]      # ambiguity allowance A
    c: Dict[str, float]
    n_ambiguous: int
    trained: Dict[str, bool] = field(default_factory=dict)


def _cells(rows: torch.Tensor, h: int, w: int):
    cell = rows % (h * w)
    return cell // w, cell % w


def shared_sample(G: torch.Tensor, cy, cx, ax, absolute=False):
    """grid_sample(G [1,C,h,w], node (cx, cy), bilinear, align_corners=True) with the fp32 node weights: [n, C] fp64,
    plus the list of (cell, weight) pairs per row for the backward."""
    _, C, h, w = G.shape
    (xi, xw0, xw1), (yi, yw0, yw1) = ax
    Gf = G.reshape(C, h * w).t().double()
    if absolute:
        Gf = Gf.abs()
    out = torch.zeros(cy.shape[0], C, dtype=torch.float64)
    taps = []
    for dy in (0, 1):
        for dx in (0, 1):
            yy, xx = yi[cy] + dy, xi[cx] + dx
            wt = (yw1[cy] if dy else yw0[cy]) * (xw1[cx] if dx else xw0[cx])
            ok = (yy < h) & (xx < w) & (wt != 0)
            cell = torch.where(ok, yy * w + xx, torch.zeros_like(yy))
            wt = torch.where(ok, wt, torch.zeros_like(wt))
            out += wt[:, None] * Gf[cell]
            taps.append((cell, wt))
    return out, taps


def encode(table: torch.Tensor, coords: torch.Tensor, meta: HG.GridMeta, absolute=False):
    """Hash-grid encoding in fp64 with the fp32 corners / weights; also returns the corners for the backward."""
    F_ = meta.n_features
    t = table.reshape(-1, F_).double()
    if absolute:
        t = t.abs()
    outs, corners = [], []
    for l in range(meta.n_levels):
        idx, wt = HG.corner_indices_weights(coords, meta, l)
        idx = idx + int(meta.offset[l])
        wt = wt.double()
        outs.append((t[idx] * wt.unsqueeze(-1)).sum(1))
        corners.append((idx, wt))
    return torch.cat(outs, 1), corners


def _relu_fwd(z, zE, zB):
    """ReLU with its envelope.  zB: a running bound of z's fp32 error (the stage's own rounding on the actual |inputs|
    plus the inputs' bounds carried through |W|); elements with |z| <= zB are ambiguous and keep their envelope."""
    amb = z.abs() <= zB
    keep = (z > 0) | amb
    return z.clamp_min(0), torch.where(keep, zE, torch.zeros_like(zE)), amb, keep


def _bound(x, xB, W, b, c):
    """Running error bound of x W^T + b: c u (|x| |W|^T + |b|), plus the inputs' bounds xB carried through W in
    quadrature (the rounding errors of different inputs are independent, as in the composition rule above)."""
    W = W.double()
    out = c * U * (x.abs() @ W.abs().t() + b.double().abs())
    return out if xB is None else out + (xB * xB @ (W * W).t()).sqrt()


def linear_env(x, xE, W, b):
    """x W^T + b and its envelope |x|_E |W|^T + |b|."""
    W, b = W.double(), b.double()
    return x @ W.t() + b, xE @ W.abs().t() + b.abs()


def field_forward(p, coords, meta, simt=False):
    enc, corners = encode(p["table"], coords, meta)
    encE, _ = encode(p["table"], coords, meta, absolute=True)
    Lf, H1 = enc.shape[1], p["mlp.0.weight"].shape[0]
    c_z1 = quad(8.0, c_gemm(Lf, simt))
    z1, z1E = linear_env(enc, encE, p["mlp.0.weight"], p["mlp.0.bias"])
    z1B = _bound(enc, 8.0 * U * encE, p["mlp.0.weight"], p["mlp.0.bias"], c_gemm(Lf, simt))
    h1, h1E, amb1, keep1 = _relu_fwd(z1, z1E, z1B)
    F, FE = linear_env(h1, h1E, p["mlp.2.weight"], p["mlp.2.bias"])
    FB = _bound(h1, z1B * keep1, p["mlp.2.weight"], p["mlp.2.bias"], c_gemm(H1, simt))
    return dict(enc=enc, encE=encE, corners=corners, z1=z1, z1E=z1E, h1=h1, h1E=h1E, amb1=amb1, F=F, FE=FE, FB=FB,
                c_F=quad(c_z1, c_gemm(H1, simt)), c_z1=c_z1)


def residual_forward(p, raw, simt=False):
    C, Hr = raw.shape[1], p["res.0.weight"].shape[0]
    c_r1 = c_gemm(C, simt)
    z1, z1E = linear_env(raw, raw.abs(), p["res.0.weight"], p["res.0.bias"])
    z1B = _bound(raw, None, p["res.0.weight"], p["res.0.bias"], c_r1)
    r1, r1E, a1, k1 = _relu_fwd(z1, z1E, z1B)
    c_r2 = quad(c_r1, c_gemm(Hr, simt))
    z2, z2E = linear_env(r1, r1E, p["res.2.weight"], p["res.2.bias"])
    z2B = _bound(r1, z1B * k1, p["res.2.weight"], p["res.2.bias"], c_gemm(Hr, simt))
    r2, r2E, a2, k2 = _relu_fwd(z2, z2E, z2B)
    q, qE = linear_env(r2, r2E, p["res.4.weight"], p["res.4.bias"])
    qB = _bound(r2, z2B * k2, p["res.4.weight"], p["res.4.bias"], c_gemm(Hr, simt))
    return dict(z1=z1, z1E=z1E, r1=r1, r1E=r1E, a1=a1, z2=z2, z2E=z2E, r2=r2, r2E=r2E, a2=a2, q=q, qE=qE, qB=qB,
                c_r1=c_r1, c_r2=c_r2, c_q=quad(c_r2, c_gemm(Hr, simt)))


def _ones(x):
    return torch.cat([x, torch.ones(x.shape[0], 1, dtype=x.dtype)], 1)


def _wgrad(dY, X):
    """dY^T [X | 1] split into (weight, bias)."""
    full = dY.t() @ _ones(X)
    return full[:, :-1].contiguous(), full[:, -1].contiguous()


def step(p: Dict[str, torch.Tensor], feats: torch.Tensor, coords: torch.Tensor, rows: torch.Tensor, h: int, w: int,
         meta: HG.GridMeta, sc: Scalars, *, exact_grid: bool = True, simt: bool = False) -> StepResult:
    """One fit step at parameters p (fp32 tensors, reference layouts).  feats [R, C], coords [R, 2] fp32: the flattened
    bank; rows: the bank rows of the step."""
    rows = torch.as_tensor(rows, dtype=torch.int64)
    raw = feats[rows].double()
    pc = coords[rows].float()
    n, C = raw.shape
    H1, Hr = C // 2, C // 4
    ls = float(sc.loss_scale)
    ax = (axis_tables(w, exact_grid), axis_tables(h, exact_grid))
    cy, cx = _cells(rows, h, w)
    # ---- forward ----
    fw = field_forward(p, pc, meta, simt)
    shared, taps = shared_sample(p["G"], cy, cx, ax)
    sharedE, _ = shared_sample(p["G"], cy, cx, ax, absolute=True)
    pred, predE, c_pred = fw["F"] + shared, fw["FE"] + sharedE, fw["c_F"]
    rs = None
    if sc.phase2:
        rs = residual_forward(p, raw, simt)
        pred, predE, c_pred = pred + rs["q"], predE + rs["qE"], max(c_pred, rs["c_q"])
    c_pred = quad(c_pred, 4.0)
    # ---- loss ----
    d = pred - raw
    np_ = pred.norm(dim=1).clamp_min(1e-8)
    nr_ = raw.norm(dim=1).clamp_min(1e-8)
    dot = (pred * raw).sum(1)
    cos = dot / (np_ * nr_)
    l2 = (d * d).mean()
    lc = 1.0 - cos.mean()
    losses = {"patch_l2_loss": float(l2), "cosine_similarity_loss": float(lc), "residual_loss": 0.0,
              "residual_sparsity_loss": 0.0}
    if sc.phase2:
        losses["residual_loss"] = float(0.1 * (d * d).mean())
        losses["residual_sparsity_loss"] = float(0.02 * rs["q"].abs().mean())
    losses["loss"] = sum(losses[k] for k in ("patch_l2_loss", "cosine_similarity_loss", "residual_loss",
                                             "residual_sparsity_loss"))
    # bounds of the logged fp32 losses: sums of nonnegative terms (per-lane C / 32 terms, 5 shuffle levels, 8 warps, n / 8
    # float atomics in arrival order) with the worst-case bound depth * u relative to the sum (~2e-5 at C = 1536), plus
    # pred's running error bound carried linearly through each term.  (Not in quadrature: after the residual MLP's first
    # Adam step its weights have moved along the gradient, so R's rounding errors correlate with pred - raw and do not
    # average out -- measured at C >= 1024, where the quadrature estimate is exceeded twofold.)
    c_red = 4.0 + C // 32 + 13 + n // 8
    e_pred = fw["FB"] + 4 * U * (sharedE + pred.abs()) + (rs["qB"] if sc.phase2 else 0)   # running bound of pred
    dcos = (raw / (np_ * nr_)[:, None] - (cos / np_ ** 2)[:, None] * pred).abs()   # |d cos / d pred|
    loss_tol = {"patch_l2_loss": c_red * U * float(l2) + float((2 * d.abs() * e_pred).mean()),
                "cosine_similarity_loss": c_red * U * (float(lc) + 1.0) + float((e_pred * dcos).sum(1).mean()),
                "residual_loss": 0.0, "residual_sparsity_loss": 0.0}
    if sc.phase2:
        loss_tol["residual_loss"] = 0.1 * loss_tol["patch_l2_loss"]
        loss_tol["residual_sparsity_loss"] = c_red * U * losses["residual_sparsity_loss"] + 0.02 * float(rs["qB"].mean())
    loss_tol["loss"] = sum(loss_tol.values())
    # ---- d pred (and its envelope: the formula on absolute values, with the norms' sensitivity to pred's error) ----
    k_mse = 2.0 * ls / (n * C)
    dpred = k_mse * d + (ls / n) * (-raw / (np_ * nr_)[:, None] + (cos / np_ ** 2)[:, None] * pred)
    rho = (predE.norm(dim=1) / np_)[:, None]
    cosE = ((predE * raw.abs()).sum(1) / (np_ * nr_))[:, None]
    dpredE = k_mse * (predE + raw.abs()) + (ls / n) * (raw.abs() / (np_ * nr_)[:, None] * (1 + rho)
                                                      + (cosE * predE + 2 * rho * cos.abs()[:, None] * pred.abs())
                                                      / (np_ ** 2)[:, None])
    c_dpred = quad(c_pred, c_sum(C // 32 + 5), 8.0)
    grad, env, allow, cc = {}, {}, {}, {}
    # ---- field MLP ----
    W1, W2 = p["mlp.0.weight"].double(), p["mlp.2.weight"].double()
    grad["mlp.2.weight"], grad["mlp.2.bias"] = _wgrad(dpred, fw["h1"])
    env["mlp.2.weight"], env["mlp.2.bias"] = _wgrad(dpredE, fw["h1E"])
    cc["mlp.2.weight"] = cc["mlp.2.bias"] = quad(c_dpred, fw["c_z1"], c_gemm(n, simt))
    u1 = dpred @ W2                      # d h1 before the mask
    u1E = dpredE @ W2.abs()
    mask1 = fw["z1"] > 0
    dh1, dh1E = u1 * mask1, torch.where(mask1 | fw["amb1"], u1E, torch.zeros_like(u1E))
    c_dh1 = quad(c_dpred, c_gemm(C, simt))
    grad["mlp.0.weight"], grad["mlp.0.bias"] = _wgrad(dh1, fw["enc"])
    env["mlp.0.weight"], env["mlp.0.bias"] = _wgrad(dh1E, fw["encE"])
    cc["mlp.0.weight"] = cc["mlp.0.bias"] = quad(c_dh1, 8.0, c_gemm(n, simt))
    # ambiguity of the field ReLU: the mask may flip -> d h1 changes by |u1| there, h1 by |z1|
    A_dh1 = torch.where(fw["amb1"], u1.abs() + U * u1E, torch.zeros_like(u1))
    Z1 = torch.where(fw["amb1"], fw["z1"].abs(), torch.zeros_like(u1))
    allow["mlp.0.weight"], allow["mlp.0.bias"] = _wgrad(A_dh1, fw["encE"])
    aw2 = dpredE.t() @ Z1
    allow["mlp.2.weight"], allow["mlp.2.bias"] = aw2, torch.zeros(C, dtype=torch.float64)
    n_amb = int(fw["amb1"].sum())
    # ---- table: d enc = d h1 W1, scattered to the corners ----
    denc, dencE, A_denc = dh1 @ W1, dh1E @ W1.abs(), A_dh1 @ W1.abs()
    c_tab = quad(c_dh1, c_gemm(H1, simt), c_sum(4 * n), 4.0)
    F_ = meta.n_features
    gt = torch.zeros(meta.n_entries, F_, dtype=torch.float64)
    gtE, gtA = torch.zeros_like(gt), torch.zeros_like(gt)
    for l, (idx, wt) in enumerate(fw["corners"]):
        sl = slice(l * F_, (l + 1) * F_)
        for k in range(4):
            gt.index_add_(0, idx[:, k], wt[:, k, None] * denc[:, sl])
            gtE.index_add_(0, idx[:, k], wt[:, k, None] * dencE[:, sl])
            gtA.index_add_(0, idx[:, k], wt[:, k, None] * A_denc[:, sl])
    grad["table"], env["table"], allow["table"], cc["table"] = gt.reshape(-1), gtE.reshape(-1), gtA.reshape(-1), c_tab
    # ---- G (phase 1 only): grid_sample backward over the four taps, neighbour shares included ----
    if not sc.phase2:
        gG = torch.zeros(h * w, C, dtype=torch.float64)
        gGE = torch.zeros_like(gG)
        for cell, wt in taps:
            gG.index_add_(0, cell, wt[:, None] * dpred)
            gGE.index_add_(0, cell, wt[:, None] * dpredE)
        grad["G"] = gG.t().reshape(1, C, h, w)
        env["G"] = gGE.t().reshape(1, C, h, w)
        allow["G"] = torch.zeros_like(grad["G"])
        cc["G"] = quad(c_dpred, c_sum(n))
    # ---- residual MLP (phase 2): e = pred - raw, d R = 0.2/(nC) ls e + 0.02/(nC) ls sign(q) ----
    if sc.phase2:
        k1, k2 = 0.2 * ls / (n * C), 0.02 * ls / (n * C)
        q = rs["q"]
        dR = k1 * d + k2 * torch.sign(q)
        dRE = k1 * (predE + raw.abs()) + k2 * (q != 0)
        c_dR = quad(c_pred, 4.0)
        ambq = q.abs() <= rs["qB"] + 4 * U * pred.abs()
        A_dR = torch.where(ambq, torch.full_like(q, 2 * k2), torch.zeros_like(q))
        dRE = torch.where(ambq, dRE + k2, dRE)
        R2, R3 = p["res.2.weight"].double(), p["res.4.weight"].double()
        grad["res.4.weight"], grad["res.4.bias"] = _wgrad(dR, rs["r2"])
        env["res.4.weight"], env["res.4.bias"] = _wgrad(dRE, rs["r2E"])
        Z2 = torch.where(rs["a2"], rs["z2"].abs(), torch.zeros_like(rs["z2"]))
        aw, ab = _wgrad(A_dR, rs["r2E"])
        allow["res.4.weight"], allow["res.4.bias"] = aw + dRE.t() @ Z2, ab
        cc["res.4.weight"] = cc["res.4.bias"] = quad(c_dR, rs["c_r2"], c_gemm(n, simt))
        # dr2 = (dR R3) * (z2 > 0)
        u2, u2E, Au2 = dR @ R3, dRE @ R3.abs(), A_dR @ R3.abs()
        m2, a2 = rs["z2"] > 0, rs["a2"]
        dr2 = u2 * m2
        dr2E = torch.where(m2 | a2, u2E, torch.zeros_like(u2E))
        A_dr2 = torch.where(m2 | a2, Au2, torch.zeros_like(Au2)) + torch.where(a2, u2.abs() + U * u2E, torch.zeros_like(u2))
        c_dr2 = quad(c_dR, c_gemm(C, simt))
        grad["res.2.weight"], grad["res.2.bias"] = _wgrad(dr2, rs["r1"])
        env["res.2.weight"], env["res.2.bias"] = _wgrad(dr2E, rs["r1E"])
        Z1r = torch.where(rs["a1"], rs["z1"].abs(), torch.zeros_like(rs["z1"]))
        aw, ab = _wgrad(A_dr2, rs["r1E"])
        allow["res.2.weight"], allow["res.2.bias"] = aw + dr2E.t() @ Z1r, ab
        cc["res.2.weight"] = cc["res.2.bias"] = quad(c_dr2, rs["c_r1"], c_gemm(n, simt))
        # dr1 = (dr2 R2) * (z1 > 0)
        R2a = R2.abs()
        u3, u3E, Au3 = dr2 @ R2, dr2E @ R2a, A_dr2 @ R2a
        m1, a1 = rs["z1"] > 0, rs["a1"]
        dr1 = u3 * m1
        dr1E = torch.where(m1 | a1, u3E, torch.zeros_like(u3E))
        A_dr1 = torch.where(m1 | a1, Au3, torch.zeros_like(Au3)) + torch.where(a1, u3.abs() + U * u3E, torch.zeros_like(u3))
        grad["res.0.weight"], grad["res.0.bias"] = _wgrad(dr1, raw)
        env["res.0.weight"], env["res.0.bias"] = _wgrad(dr1E, raw.abs())
        allow["res.0.weight"], allow["res.0.bias"] = _wgrad(A_dr1, raw.abs())
        cc["res.0.weight"] = cc["res.0.bias"] = quad(c_dr2, c_gemm(Hr, simt), c_gemm(n, simt))
        n_amb += int(ambq.sum() + rs["a1"].sum() + rs["a2"].sum())
    trained = {k: (k != "G" or not sc.phase2) and (k not in RESIDUAL or sc.phase2) for k in OF.PARAM_ORDER}
    shapes = {k: p[k].shape for k in OF.PARAM_ORDER}
    for k in grad:
        grad[k], env[k], allow[k] = grad[k].reshape(shapes[k]), env[k].reshape(shapes[k]), allow[k].reshape(shapes[k])
    return StepResult(losses, loss_tol, grad, env, allow, cc, n_amb, trained)


# ---- Adam -----------------------------------------------------------------------------------------------------------
def adam(p, m, v, g, ss, ibc, wd):
    """torch.optim.Adam (L2 decay folded in, betas (0.9, 0.99), eps 1e-15 outside the sqrt) in fp64 on fp64 inputs;
    ss = lr / (1 - 0.9^t), ibc = 1 / sqrt(1 - 0.99^t)."""
    g = g + wd * p
    m = m + 0.1 * (g - m)
    v = 0.99 * v + 0.01 * g * g
    return p - ss * m / (v.sqrt() * ibc + 1e-15), m, v


def ulp(x: torch.Tensor) -> torch.Tensor:
    """ulp of fp32 values (of their magnitude; subnormal floor)."""
    a = x.double().abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 23)


# ---- forward checks (final query / residual) ------------------------------------------------------------------------
def query_ref(p, coords, meta, simt=False):
    """F = field(coords) with its envelope and c (ReLU ambiguity only moves F by |z| |W2| <= the envelope)."""
    fw = field_forward(p, coords.float(), meta, simt)
    return fw["F"], fw["FE"], fw["c_F"]


def residual_ref(p, raw, simt=False):
    rs = residual_forward(p, raw.double(), simt)
    return rs["q"], rs["qE"], rs["c_q"]
