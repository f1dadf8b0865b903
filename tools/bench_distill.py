#!/usr/bin/env python
"""Stage-3 distillation step (reference main_distillation.py:209-249) on synthetic images: teacher forward (frozen ViT +
denoiser block), student forward, backward through the whole student ViT, gradient all-reduce + AdamW.  Default: ViT-B/14
(DINOv2 layout with LayerScale, random weights), 518 x 518, batch 32 per GPU.

Reports images/s, CUDA-event spans of the four phases, peak memory (torch.cuda.max_memory_allocated) with and without
gradient checkpointing, algorithmic FLOPs from the shapes and the TFLOP/s they imply against the data-sheet bf16 dense
peak of the H100 SXM (989 TFLOP/s), and a "library bar": the same step with torch modules (autograd, bf16 autocast,
F.scaled_dot_product_attention, cuBLAS, torch.optim.AdamW(fused=True)) -- the modules of tools/library_bar.py.  For the
SwiGLU backbones (ViT-g/14) the comparison is a torch step of the same SwiGLU model built here (SwiGLUPacked MLP,
LayerScale, torch.utils.checkpoint around every block when the checkpointed arm runs), reported as "torch_swiglu_step".
`--arms plain|ckpt` runs one of the two arms only (ViT-g at batch 32 and 518 x 518 does not fit without checkpointing).

  python tools/bench_distill.py [--steps 10 --warmup 3 --batch 32 --size 518]
  python tools/bench_distill.py --model vit_giant_patch14_dinov2.lvd142m --arms ckpt
  python -m torch.distributed.run --nproc-per-node N --master-addr 127.0.0.1 tools/bench_distill.py ...
One JSON line on rank 0.  Writes nothing to the tree."""
import argparse
import json
import os
import re
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "denoising-vit_b200"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)

PEAK_BF16_TFLOPS = 989.0   # H100 SXM data sheet, dense bf16, 700 W


def _gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else torch.cuda.get_device_name()
    except Exception:
        return torch.cuda.get_device_name()


def vit_flops(B, np_, prefix, C, depth, mlp, K, swiglu=False):
    """Algorithmic forward FLOPs (2 M N K per GEMM, 4 B N^2 C for the two attention products).  swiglu: fc1 is C -> mlp,
    fc2 is mlp / 2 -> C (timm SwiGLUPacked)."""
    N = np_ + prefix
    M = B * N
    fc2_in = mlp // 2 if swiglu else mlp
    per_block = 2 * M * C * (3 * C + C) + 2 * M * C * (mlp + fc2_in) + 4 * B * N * N * C
    return 2 * B * np_ * K * C + depth * per_block


def _torch_swiglu_student(C, depth, heads, P, grid, mlp, ckpt):
    """Torch comparison model for the SwiGLU backbones: tools/library_bar.py's ViT with timm SwiGLUPacked MLPs ([g | u] =
    fc1(x), fc2(silu(g) * u)), SDPA attention, LayerScale, and torch.utils.checkpoint around every block when `ckpt`."""
    import library_bar
    from torch import nn
    from torch.utils.checkpoint import checkpoint

    class Block(library_bar._Block):
        def __init__(self):
            super().__init__(C, heads)
            self.fc1, self.fc2 = nn.Linear(C, mlp), nn.Linear(mlp // 2, C)

        def forward(self, x):
            B, N, _ = x.shape
            q, k, v = self.qkv(self.n1(x)).reshape(B, N, 3, self.heads, C // self.heads).permute(2, 0, 3, 1, 4).unbind(0)
            x = x + self.g1 * self.proj(F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, N, C))
            g, u = self.fc1(self.n2(x)).chunk(2, dim=-1)
            return x + self.g2 * self.fc2(F.silu(g) * u)

    class ViT(library_bar._ViT):
        def __init__(self):
            super().__init__(C, 0, heads, P, grid)
            self.blocks = nn.ModuleList([Block() for _ in range(depth)])

        def forward(self, x):
            x = self.patch(x).flatten(2).transpose(1, 2)
            x = torch.cat([self.cls.expand(x.shape[0], -1, -1), x], 1) + self.pos
            for b in self.blocks:
                x = checkpoint(b, x, use_reentrant=False) if (ckpt and torch.is_grad_enabled()) else b(x)
            return self.norm(x)[:, 1:]

    return ViT()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="vit_base_patch14_dinov2.lvd142m")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--size", type=int, default=518)
    ap.add_argument("--no-library", action="store_true")
    ap.add_argument("--arms", choices=("both", "plain", "ckpt"), default="both",
                    help="run the plain step, the gradient-checkpointed step or both (ViT-g at batch 32 and 518 x 518 only "
                         "fits with checkpointing)")
    ap.add_argument("--deterministic", action="store_true",
                    help="torch.use_deterministic_algorithms(True): the fixed-order backward kernels")
    ap.add_argument("--no-empty-fill", action="store_true",
                    help="with --deterministic: skip torch's NaN fill of torch.empty (measures what that fill costs)")
    a = ap.parse_args()
    if a.deterministic:
        torch.use_deterministic_algorithms(True)
        if a.no_empty_fill:
            torch.utils.deterministic.fill_uninitialized_memory = False
        print(f"deterministic mode (NaN fill of empty tensors: {not a.no_empty_fill})")
    rank, world, local = (int(os.environ.get(k, d)) for k, d in (("RANK", "0"), ("WORLD_SIZE", "1"), ("LOCAL_RANK", "0")))
    assert torch.cuda.is_available(), "bench_distill needs a CUDA device"
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=dev)
    import dvt.models as DVT
    from dvt import train_ops
    from dvt.optim import FusedAdamW

    B = a.batch
    student = DVT.PretrainedViTWrapper(a.model, stride=int(re.search(r"patch(\d+)", a.model).group(1)), allow_random_init=True).to(dev)
    P = student.patch_size
    arch = student.model.arch
    C, depth, heads, mlp, prefix = arch["embed"], arch["depth"], arch["heads"], arch["mlp"], student.model.num_prefix_tokens
    h = w = (a.size - P) // P + 1
    teacher_vit = DVT.PretrainedViTWrapper(a.model, stride=P, allow_random_init=True)
    teacher_vit.load_state_dict(student.state_dict())
    teacher = DVT.Denoiser(h, w, C, vit=teacher_vit, num_blocks=1).to(dev).eval()
    g = torch.Generator(device=dev).manual_seed(rank)
    imgs = torch.randn(B, 3, a.size, a.size, device=dev, generator=g)
    student.set_trainable(True)
    opt = FusedAdamW(student.parameters(), lr=1e-5, betas=(0.9, 0.999), weight_decay=1e-5)

    ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
    spans = []

    def step(record):
        ev[0].record()
        with torch.no_grad():
            target = teacher(imgs, return_dict=True)["denoised_feats"]
        ev[1].record()
        pred = student.get_intermediate_layers(imgs)[0].permute(0, 2, 3, 1)
        loss, _, _ = train_ops.denoise_loss(pred, target)
        ev[2].record()
        opt.zero_grad()
        loss.backward()
        ev[3].record()
        opt.sync_grads(world)
        opt.step()
        ev[4].record()
        if record:
            torch.cuda.synchronize()
            spans.append([ev[i].elapsed_time(ev[i + 1]) for i in range(4)])

    def run(ckpt):
        student.model.set_grad_checkpointing(ckpt)
        for _ in range(a.warmup):
            step(False)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        spans.clear()
        for _ in range(a.steps):
            step(True)
        sp = torch.tensor(spans).mean(0).tolist()
        return sp, torch.cuda.max_memory_allocated()

    phases = ("teacher_fwd", "student_fwd", "backward", "allreduce_adamw")
    sp, mem = run(False) if a.arms != "ckpt" else (None, None)
    sp_ck, mem_ck = run(True) if a.arms != "plain" else (None, None)
    np_ = h * w
    K = 3 * P * P
    swiglu = bool(arch["swiglu"])
    f_vit = vit_flops(B, np_, prefix, C, depth, mlp, K, swiglu)
    f_den = vit_flops(B, np_, 0, C, 1, 4 * C, 0)
    flops = f_vit + f_den + 3 * f_vit          # teacher (ViT + denoiser block) + student forward + backward (2 x forward)
    # headline: the plain step (the checkpointed one with --arms ckpt); checkpointing adds a recompute of the student
    # forward that the algorithmic FLOPs do not count
    head_sp, head_mem = (sp, mem) if sp is not None else (sp_ck, mem_ck)
    ms = sum(head_sp)
    out = {"metric": f"stage-3 distillation images/s ({a.model}, {a.size}x{a.size}, batch {B} per GPU)",
           "value": world * B * 1000.0 / ms, "unit": "images/s", "n_gpus": world, "ms_per_step": ms,
           "span_ms": dict(zip(phases, head_sp)),
           "max_memory_allocated_gb": head_mem / 2 ** 30}
    if a.arms != "both":
        out["arm"] = "grad_checkpointing" if a.arms == "ckpt" else "plain"
    if a.arms == "both":
        out["grad_checkpointing"] = {"ms_per_step": sum(sp_ck), "images_per_s": world * B * 1000.0 / sum(sp_ck),
                                     "span_ms": dict(zip(phases, sp_ck)), "max_memory_allocated_gb": mem_ck / 2 ** 30}
    out.update({"algorithmic_tflop_per_step": flops / 1e12, "tflops_per_gpu": flops / (ms / 1e3) / 1e12,
                "share_of_bf16_peak": flops / (ms / 1e3) / 1e12 / PEAK_BF16_TFLOPS,
                "dtype": "bf16 GEMMs / attention, fp32 master weights and residual stream", "data": "synthetic",
                "gpu": _gpu_info()})
    if not a.no_library and rank == 0 and swiglu:
        # torch step of the same SwiGLU model: autograd, bf16 autocast, SDPA, torch.utils.checkpoint (unless only the plain
        # arm ran), torch.optim.AdamW(fused=True); the teacher is the frozen torch ViT plus one torch block
        import gc
        import library_bar
        ckpt = a.arms != "plain"
        del opt, student, teacher, teacher_vit
        gc.collect()
        torch.cuda.empty_cache()
        with torch.device(dev):
            ref = _torch_swiglu_student(C, depth, heads, P, h, mlp, ckpt).train()
            rt_vit = _torch_swiglu_student(C, depth, heads, P, h, mlp, False).eval().requires_grad_(False)
            rt_blk = library_bar._Block(C, heads).eval().requires_grad_(False)
        ropt = torch.optim.AdamW(ref.parameters(), lr=1e-5, betas=(0.9, 0.999), weight_decay=1e-5, fused=True)

        def tstep():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                with torch.no_grad():
                    tgt = rt_blk(rt_vit(imgs)).float().reshape(B, h, w, C)
                pred = ref(imgs).float().reshape(B, h, w, C)
                loss = F.mse_loss(pred, tgt) + 1 - F.cosine_similarity(pred, tgt, dim=-1).mean()
            ropt.zero_grad()
            loss.backward()
            ropt.step()

        for _ in range(a.warmup):
            tstep()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.steps):
            tstep()
        e1.record()
        torch.cuda.synchronize()
        tms = e0.elapsed_time(e1) / a.steps
        out["torch_swiglu_step"] = {"ms_per_step": tms, "images_per_s": B * 1000.0 / tms, "grad_checkpointing": ckpt,
                                    "tflops": flops / (tms / 1e3) / 1e12,
                                    "max_memory_allocated_gb": torch.cuda.max_memory_allocated() / 2 ** 30}
    elif not a.no_library and rank == 0:
        import library_bar
        del opt
        torch.cuda.empty_cache()
        ref = library_bar._ViT(C, depth, heads, P, h).to(dev).train()
        rt_vit = library_bar._ViT(C, depth, heads, P, h).to(dev).eval()
        rt_blk = library_bar._Block(C, heads).to(dev).eval()
        rt_pos = torch.zeros(1, np_, C, device=dev)
        ropt = torch.optim.AdamW(ref.parameters(), lr=1e-5, betas=(0.9, 0.999), weight_decay=1e-5, fused=True)

        def rstep():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                with torch.no_grad():
                    tgt = rt_blk(rt_vit(imgs) + rt_pos).float().reshape(B, h, w, C)
                pred = ref(imgs).float().reshape(B, h, w, C)
                loss = F.mse_loss(pred, tgt) + 1 - F.cosine_similarity(pred, tgt, dim=-1).mean()
            ropt.zero_grad()
            loss.backward()
            ropt.step()

        for _ in range(a.warmup):
            rstep()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.steps):
            rstep()
        e1.record()
        torch.cuda.synchronize()
        rms = e0.elapsed_time(e1) / a.steps
        out["library_bar_bf16_autocast"] = {"ms_per_step": rms, "images_per_s": B * 1000.0 / rms,
                                            "max_memory_allocated_gb": torch.cuda.max_memory_allocated() / 2 ** 30}
    if rank == 0:
        print(json.dumps(out), flush=True)
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
