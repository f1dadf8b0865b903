"""GPU "library bar" (BASELINE.md section 4.5, SURVEY.md 8(d)): what the reference's own op sequence costs on the SAME
H100 when every op goes to the vendor libraries -- the number the fused kernels of this repository have to beat.

  * HP-1: a ViT-B/14 forward as the reference reaches it through timm (vit_wrapper.py:136-143): Conv2d patch embedding,
    per block LayerNorm -> Linear(qkv) -> F.scaled_dot_product_attention -> Linear(proj) -> LayerScale + residual ->
    LayerNorm -> Linear -> GELU -> Linear -> LayerScale + residual, final LayerNorm; cuDNN / cuBLAS / SDPA kernels; fp32
    (torch default, TF32 off) and bf16 autocast (the reference's `--dtype bfloat16`).
  * HP-2: one optimisation step as main_img_denoising.py:67-89 runs it: three fancy-index gathers, `F.grid_sample` for G,
    a hash-grid encoding with a DENSE table gradient (tcnn is not installable: plain index ops), two nn.Linear MLPs, the
    five loss terms, `loss * 1024`, backward, `torch.optim.Adam(foreach=True)` over all 21 M parameters.

Self-contained on purpose (plain torch modules, nothing from oracle/ and nothing from libdvt_b200): it is a baseline that
is MEASURED, not a checker.  Timed with CUDA events after warm-up; bench.py prints the result under `library_bar`."""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F


class _Block(nn.Module):
    def __init__(self, C, heads):
        super().__init__()
        self.heads = heads
        self.n1, self.n2 = nn.LayerNorm(C, eps=1e-6), nn.LayerNorm(C, eps=1e-6)
        self.qkv, self.proj = nn.Linear(C, 3 * C), nn.Linear(C, C)
        self.fc1, self.fc2 = nn.Linear(C, 4 * C), nn.Linear(4 * C, C)
        self.g1, self.g2 = nn.Parameter(torch.ones(C)), nn.Parameter(torch.ones(C))

    def forward(self, x):
        B, N, C = x.shape
        q, k, v = self.qkv(self.n1(x)).reshape(B, N, 3, self.heads, C // self.heads).permute(2, 0, 3, 1, 4).unbind(0)
        a = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, N, C)
        x = x + self.g1 * self.proj(a)
        return x + self.g2 * self.fc2(F.gelu(self.fc1(self.n2(x))))


class _ViT(nn.Module):
    def __init__(self, C=768, depth=12, heads=12, patch=14, grid=37):
        super().__init__()
        self.patch = nn.Conv2d(3, C, patch, patch)
        self.cls = nn.Parameter(torch.zeros(1, 1, C))
        self.pos = nn.Parameter(torch.randn(1, 1 + grid * grid, C) * 0.02)
        self.blocks = nn.ModuleList([_Block(C, heads) for _ in range(depth)])
        self.norm = nn.LayerNorm(C, eps=1e-6)

    def forward(self, x):
        x = self.patch(x).flatten(2).transpose(1, 2)
        x = torch.cat([self.cls.expand(x.shape[0], -1, -1), x], 1) + self.pos
        for b in self.blocks:
            x = b(x)
        return self.norm(x)[:, 1:]


def _events():
    return torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


@torch.no_grad()
def vit_forward_bar(dev, batch=32, reps=3):
    """s per 518 x 518 view of the unfused ViT-B/14 forward: fp32 and bf16 autocast."""
    model = _ViT().to(dev).eval()
    x = torch.randn(batch, 3, 518, 518, device=dev)
    out = {}
    for name, ctx in (("fp32", torch.autocast("cuda", enabled=False)), ("bf16_autocast", torch.autocast("cuda", dtype=torch.bfloat16))):
        with ctx:
            model(x)
            torch.cuda.synchronize()
            e0, e1 = _events()
            e0.record()
            for _ in range(reps):
                model(x)
            e1.record()
            torch.cuda.synchronize()
        out[name] = e0.elapsed_time(e1) / 1e3 / (reps * batch)
    return out


def _grid_levels(n_levels=16, base=16, max_res=1024, log2_hash=20):
    pls = math.exp(math.log(max_res / base) / (n_levels - 1)) if n_levels > 1 else 1.0
    lv, off = [], 0
    for l in range(n_levels):
        scale = np.float32(np.exp2(np.float32(l) * np.log2(np.float32(pls))) * np.float32(base) - np.float32(1.0))
        res = int(np.ceil(scale)) + 1
        size = min((res * res + 7) // 8 * 8, 1 << log2_hash)
        lv.append((float(scale), res, size, off, res * res > size))
        off += size
    return lv, off


def _encode(table, xy, levels):
    outs = []
    for scale, res, size, off, hashed in levels:
        pos = xy * scale + 0.5
        cell = pos.floor()
        w = pos - cell
        cx, cy = cell[:, 0].long(), cell[:, 1].long()
        acc = 0
        for dy in (0, 1):
            for dx in (0, 1):
                x, y = cx + dx, cy + dy
                idx = ((x ^ (y * 2654435761)) & 0xFFFFFFFF) % size if hashed else (x + y * res) % size
                wt = (w[:, 0] if dx else 1 - w[:, 0]) * (w[:, 1] if dy else 1 - w[:, 1])
                acc = acc + table[off + idx] * wt.unsqueeze(-1)
        outs.append(acc)
    return torch.cat(outs, -1)


def fit_step_bar(dev, C=768, h=37, w=37, V=64, bsz=2048, steps=20, warm=5):
    """s per optimisation step (phase 1, phase 2) of the unfused fit at the headline size (bank of V views)."""
    g = torch.Generator(device=dev).manual_seed(0)
    levels, entries = _grid_levels()
    table = nn.Parameter((torch.rand(entries, 8, device=dev, generator=g) * 2 - 1) * 1e-4)
    mlp = nn.Sequential(nn.Linear(128, C // 2), nn.ReLU(), nn.Linear(C // 2, C)).to(dev)
    G = nn.Parameter(torch.randn(1, C, h, w, device=dev, generator=g) * 0.02)
    res = nn.Sequential(nn.Linear(C, C // 4), nn.ReLU(), nn.Linear(C // 4, C // 4), nn.ReLU(), nn.Linear(C // 4, C)).to(dev)
    params = [G] + list(res.parameters()) + [table] + list(mlp.parameters())
    opt = torch.optim.Adam(params, lr=0.01, eps=1e-15, weight_decay=1e-5, betas=(0.9, 0.99), foreach=True)
    bank = torch.randn(V * h * w, C, device=dev, generator=g)
    coords = torch.rand(V * h * w, 2, device=dev, generator=g)
    ys, xs = torch.linspace(-1, 1, h), torch.linspace(-1, 1, w)
    gy, gx = torch.meshgrid(ys, xs, indexing="ij")
    gcoords = torch.stack([gx, gy], -1).reshape(-1, 2).repeat(V, 1).to(dev)
    rs = np.random.RandomState(0)

    def step(phase2):
        idx = rs.randint(0, bank.shape[0], bsz)                       # host indices -> 3 implicit H2D copies, like the reference
        raw, gc, pc = bank[idx], gcoords[idx], coords[idx]
        shared = F.grid_sample(G, gc[None, None], mode="bilinear", align_corners=True).squeeze().permute(1, 0)
        den = mlp(_encode(table, pc, levels))
        if phase2:
            pr = res(raw)
            pred = den + shared + pr.detach()
        else:
            pred = shared + den
        loss = F.mse_loss(pred, raw) + 1 - F.cosine_similarity(pred, raw, dim=-1).mean()
        if phase2:
            loss = loss + 0.1 * F.mse_loss(pr, (raw - den - shared).detach()) + 0.02 * pr.abs().mean()
        opt.zero_grad()
        (loss * 1024.0).backward()
        opt.step()

    out = {}
    for phase2 in (False, True):
        if phase2:
            G.requires_grad = False
        for _ in range(warm):
            step(phase2)
        torch.cuda.synchronize()
        e0, e1 = _events()
        e0.record()
        for _ in range(steps):
            step(phase2)
        e1.record()
        torch.cuda.synchronize()
        out["phase2" if phase2 else "phase1"] = e0.elapsed_time(e1) / 1e3 / steps
    return out


def measure(dev, views=769, num_iters=2000, batch=32):
    v = vit_forward_bar(dev, batch=batch)
    f = fit_step_bar(dev)
    n_p2 = num_iters - 1 - int(0.5 * num_iters)
    n_p1 = num_iters - n_p2
    fit_s = n_p1 * f["phase1"] + n_p2 * f["phase2"]
    return {"what": "the reference's op sequence on this GPU through cuDNN / cuBLAS / SDPA / ATen / torch.optim (unfused)",
            "vit_s_per_view": v, "fit_s_per_step": f, "fit_s_per_image": fit_s,
            "hp1_s_per_image": {k: views * t for k, t in v.items()},
            "images_per_s": {k: 1.0 / (views * t + fit_s) for k, t in v.items()},
            "sample": f"{3 * batch} views per precision, 20 fit steps per phase after 5 warm-up, extrapolated to "
                      f"{views} views + {num_iters} steps"}


if __name__ == "__main__":
    import json
    print(json.dumps(measure(torch.device("cuda", 0)), indent=1))
