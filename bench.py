#!/usr/bin/env python
"""Headline benchmark: images/sec of DVT stage-1 denoising (ViT-B/14, 518x518, 768+1 views, 2000-iteration
neural-field fit per image) on N H100s of one node.  One "step" = one image through both hot paths:
HP-1 769 frozen-ViT forwards -> feature bank, HP-2 per-image fit + final 37x37 query.

  python bench.py --gpus 1 --steps 3 --warmup 3
  python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P bench.py --gpus N ...
  python bench.py --impl reference ...      # the reference algorithm on the host CPU cores (oracle port), same metric

Prints ONE JSON line (rank 0).  `value` is device-resident throughput (inputs in HBM); `e2e` goes through the public
per-image call with pinned HOST views, host->device copies and device->host result reads inside the timed region.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "denoising-vit_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

MODEL = "vit_base_patch14_dinov2.lvd142m"
FLOPS_PER_VIEW = 303.1e9                 # SURVEY.md section 8(d): 1.24 + 12 x (4.85 + 5.77 + 1.62 + 12.93) GF
FIT_BYTES_P1, FIT_BYTES_P2 = 522e6, 505e6  # SURVEY.md section 8(d): algorithmic bytes per fit step (dense Adam, 24 B/param)


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", type=str, default="b200", choices=["b200", "reference"])
    ap.add_argument("--views", type=int, default=768)
    ap.add_argument("--num-iters", type=int, default=2000)
    ap.add_argument("--warmup-iters", type=int, default=200)
    ap.add_argument("--extract-bsz", type=int, default=32)
    ap.add_argument("--graph-steps", type=int, default=20)
    ap.add_argument("--no-overlap", action="store_true", help="one image strictly after the other (A/B of the schedule)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-kernel-rooflines", action="store_true",
                    help="skip the stand-alone kernel timings (for ncu launch lists of the timed region)")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--dump-outputs", type=str, default=None, metavar="DIR",
                    help="after the timed steps, write the last timed image's results (denoised_feats, raw) as DIR/<name>.npy "
                         "(float32); inputs and weights are seeded, so two builds can be compared output for output")
    ap.add_argument("--no-library-bar", action="store_true",
                    help="skip the unfused cuBLAS / SDPA / torch.optim restatement timed on the same GPU (tools/library_bar.py)")
    return ap.parse_args()


def peaks():
    """HBM copy bandwidth and dense bf16 throughput: the driver-written MEASURED_PEAKS.json (burst figure for a kernel
    timed alone, sustained one for a path timed inside a long step), else the H100 SXM data sheet (dense bf16, HBM3)."""
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.isfile(path):
        d = json.load(open(path))
        return {"hbm_gbs": d["hbm_gbs"], "bf16_tflops": d.get("bf16_tflops_sustained", d["bf16_tflops"]),
                "bf16_tflops_burst": d["bf16_tflops"], "source": "MEASURED_PEAKS.json"}
    return {"hbm_gbs": 3350.0, "bf16_tflops": 989.0, "bf16_tflops_burst": 989.0, "source": "H100 SXM data sheet"}


def kernel_rooflines(pipe, extract_bsz, dev):
    """The two kernels that dominate the step, each timed ALONE with CUDA events on the stream it is launched on
    (10 launches after 3 warm-ups, L2 flushed by a 256 MB write before every launch), through the library's unit entry
    points -- the same kernels, shapes and epilogues the timed region launches:
      * gemm_wgmma_kernel (bf16 wgmma GEMM): the four GEMMs of one ViT-B block at the extraction batch
        (QKV, out-proj + LayerScale residual, fc1 + GELU, fc2 + LayerScale residual); algorithmic flops =
        SURVEY.md 8(d) per-view figures (4.85 + 1.62 + 12.93 GF) x views per launch set;
      * fit_adam_table_kernel (dense Adam sweep of the hash table): algorithmic bytes = 24 B x 19 741 760 parameters."""
    from dvt import ops
    g = torch.Generator(device=dev).manual_seed(0)
    rn = lambda *sh: torch.randn(*sh, device=dev, generator=g)  # noqa: E731
    Bv, N, C = extract_bsz, 1370, 768
    M = Bv * N
    x, xn, hid = rn(M, C), rn(M, C).bfloat16(), rn(M, 4 * C).bfloat16()
    w_qkv, b_qkv = (rn(3 * C, C) / 28).bfloat16(), rn(3 * C)
    w_proj, b_proj = (rn(C, C) / 28).bfloat16(), rn(C)
    w_fc1, b_fc1 = (rn(4 * C, C) / 28).bfloat16(), rn(4 * C)
    w_fc2, b_fc2 = (rn(C, 4 * C) / 55).bfloat16(), rn(C)
    gam = torch.full((C,), 1e-3, device=dev)
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
    gemms = [lambda: ops.gemm_tn(xn, w_qkv, b_qkv, None, torch.bfloat16),
             lambda: ops.gemm_tn_residual_(x, xn, w_proj, b_proj, gam),
             lambda: ops.gemm_tn(xn, w_fc1, b_fc1, "gelu", torch.bfloat16),
             lambda: ops.gemm_tn_residual_(x, hid, w_fc2, b_fc2, gam)]

    def time_alone(fn, reps=10, warm=3):
        for _ in range(warm):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(reps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        return float(np.mean(ts))

    gemm_ms = [time_alone(fn) for fn in gemms]
    gemm_flops = Bv * (4.85e9 + 1.62e9 + 12.93e9)
    sweep_ctas = int(os.environ.get("DVT_FIT_SWEEP_CTAS", "48").split(",")[0])  # geometry of the timed region (fit.cu default)
    del flush

    def time_stream(fn, reps=20, warm=3):
        """20 back-to-back launches between one event pair (the queue stays full, so host launch latency is not in the
        figure); no flush: the sweep streams 474 MB per launch, far more than the L2 holds."""
        for _ in range(warm):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps

    sweep_ms = time_stream(lambda: pipe.engine.sweep_once(max(sweep_ctas, 0)))
    sweep_full_ms = time_stream(lambda: pipe.engine.sweep_once(0))
    sweep_bytes = 24.0 * pipe.field.neural_field.params.numel()
    gbs = lambda ms: sweep_bytes / (ms / 1e3) / 1e9  # noqa: E731
    return {"gemm_ms": gemm_ms, "gemm_tflops": gemm_flops / (sum(gemm_ms) / 1e3) / 1e12, "gemm_flops": gemm_flops,
            "sweep_ms": sweep_ms, "sweep_gbs": gbs(sweep_ms), "sweep_bytes": sweep_bytes, "sweep_ctas": sweep_ctas,
            "sweep_full_ms": sweep_full_ms, "sweep_full_gbs": gbs(sweep_full_ms)}


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled every 200 ms during the timed region."""
    Q = ("clocks.sm,clocks.max.sm,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index: int):
        self.rows, self.proc, self.index = [], None, index

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms",
                                          "200", "-i", str(self.index)], stdout=subprocess.PIPE, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        sm = [float(r[0]) for r in self.rows if len(r) >= 6 and r[0].replace(".", "").isdigit()]
        mx = [float(r[1]) for r in self.rows if len(r) >= 6 and r[1].replace(".", "").isdigit()]
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        reasons = [n for j, n in enumerate(names) if any(len(r) >= 6 and r[2 + j].lower().startswith("active") for r in self.rows)]
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": reasons, "samples": len(sm)}


# ------------------------------------------------------------------------------------------------------------
# CPU arm: the reference algorithm (oracle port, fp32 PyTorch CPU) on a bounded sample, extrapolated per image
# ------------------------------------------------------------------------------------------------------------
def usable_cpus() -> int:
    """CPUs this process may actually use: affinity mask capped by the cgroup CPU quota (a container that sees 128
    logical CPUs but is limited to a few cores thrashes when given 128 threads)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        quota, period = open("/sys/fs/cgroup/cpu.max").read().split()
        if quota != "max":
            n = min(n, max(1, int(float(quota) / float(period))))
    except Exception:
        pass
    return max(1, n)


def workload_config(args, world: int) -> dict:
    """`config` of the JSON line -- identical for the GPU arm and the reference arm (same workload, same sizes)."""
    return {"workload": "stage1_vitb14_518_768views_2000iters", "views_per_image": args.views + 1,
            "fit_iters": args.num_iters, "fit_warmup_iters": args.warmup_iters, "pixel_bsz": 2048, "n_levels": 16,
            "extract_bsz": args.extract_bsz, "images_per_gpu": args.steps,
            "parallelism": f"image-sharded x{world}, one all-gather of denoised maps",
            "l2": "inputs larger than L2 (2.48 GB of views, 3.2 GB bank, 0.34 GB Adam state per image)"}


class CpuReference:
    """The reference algorithm on the host cores (oracle port, fp32 PyTorch CPU).  Built once (ViT-B/14 weights, the
    19.7 M-entry table, a small synthetic bank); every `measure()` times a bounded sample of the per-image work:
    `views_sample` ViT-B/14 forwards at 518^2 and `fit_steps` full-size optimisation steps per phase (one extra warm-up
    step per phase is not timed), and extrapolates to 769 views + 2000 steps."""

    def __init__(self, args):
        from oracle import fit as OF
        from oracle import hashgrid as HG
        from oracle import vit as OV
        self.args, self.OF, self.OV = args, OF, OV
        self.cores = min(usable_cpus(), 32)  # measured on the GPU box: 128 threads run these ops ~100x slower than 8-32 do
        torch.set_num_threads(self.cores)
        self.cfg = OV.CONFIGS[MODEL]
        self.sd = OV.random_state_dict(self.cfg, seed=0)
        self.x = torch.randn(1, 3, 518, 518, generator=torch.Generator().manual_seed(0))
        OV.forward_intermediates(self.sd, self.cfg, self.x, [11])  # warm-up
        # fit steps at the full problem size (C 768, 37x37, 16 levels, 2048 pixels); small synthetic bank of 8 views
        C, h, w, V = 768, 37, 37, 8
        self.meta = HG.grid_meta(16)
        feats, coords = OF.synthetic_bank(V, h, w, C, seed=0)
        self.init = OF.init_params(C, h, w, self.meta, seed=0)
        self.g_all = OF.make_patch_coordinates(h, w).unsqueeze(0).repeat(V, 1, 1, 1).reshape(-1, 2)
        self.f2, self.c2 = feats.reshape(-1, C), coords.reshape(-1, 2)
        self.rs = np.random.RandomState(0)

    def measure(self, views_sample: int = 1, fit_steps: int = 2):
        OF, args = self.OF, self.args
        t0 = time.perf_counter()
        for _ in range(views_sample):
            self.OV.forward_intermediates(self.sd, self.cfg, self.x, [11])
        t_view = (time.perf_counter() - t0) / views_sample
        T = 2 * fit_steps + 2
        idx = self.rs.randint(0, self.f2.shape[0], (T, 2048))
        p = {k: self.init[k].clone().float().requires_grad_(True) for k in OF.PARAM_ORDER}
        opt = torch.optim.Adam([p[k] for k in OF.PARAM_ORDER], lr=0.01, eps=1e-15, weight_decay=1e-5, betas=(0.9, 0.99))
        times = {False: [], True: []}
        for step in range(T):
            phase2 = step > T // 2
            if phase2:
                p["G"].requires_grad = False
            t0 = time.perf_counter()
            i = torch.from_numpy(idx[step])
            out = OF.denoiser_forward(p, self.f2[i], self.c2[i], self.meta, self.g_all[i], phase2)
            opt.zero_grad()
            (out["loss"] * 1024.0).backward()
            opt.step()
            dt = time.perf_counter() - t0
            if step not in (0, T // 2 + 1):  # first step of each phase = warm-up
                times[phase2].append(dt)
        assert times[False] and times[True], "CpuReference.measure: fit_steps must be >= 2 (one timed step per phase)"
        t_p1, t_p2 = float(np.mean(times[False])), float(np.mean(times[True]))
        n_p2 = args.num_iters - 1 - int(0.5 * args.num_iters)
        n_p1 = args.num_iters - n_p2
        per_image = (args.views + 1) * t_view + n_p1 * t_p1 + n_p2 * t_p2
        return {"value": 1.0 / per_image, "unit": "images/s", "cores": self.cores, "kind": "port",
                "sample": (f"{views_sample} ViT-B/14 518^2 forwards ({t_view:.3f} s/view) + {len(times[False])}+{len(times[True])} "
                           f"full-size fit steps ({t_p1:.3f} / {t_p2:.3f} s/step phase 1/2), extrapolated to "
                           f"{args.views + 1} views + {args.num_iters} steps"),
                "s_per_view": t_view, "s_per_step_phase1": t_p1, "s_per_step_phase2": t_p2}


def cpu_reference_rate(args, views_sample: int = 4, fit_steps: int = 10):
    """`cpu_baseline` of the GPU line: ~10-30 s of CPU work (4 views, 10 + 10 timed steps)."""
    return CpuReference(args).measure(views_sample, fit_steps)


def run_reference_arm(args, rank):
    """--impl reference: every "step" is a bounded sample of one image's work on the host cores, sized so that the whole
    --steps K --warmup W run ends within a few minutes (the full per-image CPU run is ~14 min): the per-step sample shrinks
    as K grows, never below 2 views + 4 timed steps per phase."""
    if rank != 0:
        return
    ref = CpuReference(args)
    n_meas = max(1, args.warmup > 0) + args.steps
    budget = 150.0 / n_meas                                   # seconds of CPU work per step
    views_sample = int(min(4, max(2, budget * 0.25 / 0.65)))
    fit_steps = int(min(10, max(4, budget * 0.75 / 0.8)))
    vals, last = [], None
    for _ in range(n_meas):
        t0 = time.perf_counter()
        last = ref.measure(views_sample=views_sample, fit_steps=fit_steps)
        vals.append((last["value"], time.perf_counter() - t0))
    vals = vals[1:] if len(vals) > 1 else vals
    v = float(np.mean([a for a, _ in vals]))
    last["value"] = v
    line = {"metric": "images/sec stage-1 denoise (ViT-B/14, 518^2, 2k-iter fit)", "value": v, "unit": "images/s",
            "impl": "reference", "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": 1000.0 / v, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
            "data": "synthetic",
            "config": workload_config(args, args.gpus),
            "arm_notes": "reference algorithm (oracle port, PyTorch CPU fp32) on a bounded sample per step, extrapolated to "
                         "one image; rank 0 only",
            "cpu_baseline": last,
            "e2e": {"value": v, "unit": "images/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line))


# ------------------------------------------------------------------------------------------------------------
# GPU arm
# ------------------------------------------------------------------------------------------------------------
def synthetic_coords(V, h, w, seed, device):
    """Seeded crop-box stream (scale in [0.1, 0.5], ratio in [3/4, 4/3], p(flip) = 0.5) -> patch coordinates in [0,1];
    last view = full image (main_img_denoising.py:288-294,337)."""
    rs = np.random.RandomState(seed)
    out = torch.zeros(V, h, w, 2)
    for v in range(V - 1):
        area = rs.uniform(0.1, 0.5)
        ratio = np.exp(rs.uniform(np.log(3 / 4), np.log(4 / 3)))
        cw, ch = min(1.0, np.sqrt(area * ratio)), min(1.0, np.sqrt(area / ratio))
        x0, y0 = rs.uniform(0, 1 - cw), rs.uniform(0, 1 - ch)
        xs, ys = torch.linspace(x0, x0 + cw, w), torch.linspace(y0, y0 + ch, h)
        if rs.rand() < 0.5:
            xs = xs.flip(0)
        gy, gx = torch.meshgrid(ys, xs, indexing="ij")
        out[v] = torch.stack([gx, gy], -1)
    ys, xs = torch.linspace(0, 1, h), torch.linspace(0, 1, w)
    gy, gx = torch.meshgrid(ys, xs, indexing="ij")
    out[-1] = torch.stack([gx, gy], -1)
    return out.clamp_(0, 1).to(device)


def main():
    args = parse()
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if args.impl == "reference":
        run_reference_arm(args, rank)
        return

    import torch.distributed as dist

    import dvt.models as DVT
    from dvt import _lib
    from dvt.stage1 import Stage1Config, Stage1Pipeline

    assert torch.cuda.is_available(), "bench.py needs a CUDA device (no CPU fallback); use --impl reference for the CPU arm"
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        # NCCL prints its version banner on STDOUT at NCCL_DEBUG=VERSION/INFO; stdout must carry the one JSON line only
        if os.environ.get("NCCL_DEBUG", "").upper() in ("VERSION", "INFO", "TRACE"):
            os.environ.setdefault("NCCL_DEBUG_FILE", "/tmp/nccl_debug.%h.%p.log")
        dist.init_process_group("nccl", device_id=dev)

    V = args.views + 1
    torch.manual_seed(0)  # the randomly initialised ViT: identical weights from run to run
    vit = DVT.PretrainedViTWrapper(MODEL, stride=14, allow_random_init=True)
    with torch.no_grad():
        for b in vit.model.blocks:  # non-degenerate LayerScale (DINOv2 init 1e-5 would switch the blocks off)
            b.ls1.gamma.fill_(1.0)
            b.ls2.gamma.fill_(1.0)
    vit = vit.to(dev).eval()
    cfg = Stage1Config(num_iters=args.num_iters, warmup_iters=args.warmup_iters, n_levels=16, extract_bsz=args.extract_bsz,
                       pixel_bsz=2048, graph_steps=args.graph_steps,
                       fit_engines=int(os.environ.get("DVT_FIT_ENGINES", Stage1Config.fit_engines)))
    pipe = Stage1Pipeline(vit, layer_index=11, input_size=(518, 518), cfg=cfg)
    h, w, C = pipe.h, pipe.w, pipe.C

    # synthetic inputs: views larger than L2 (2.48 GB fp32), host copy pinned for the e2e leg
    g = torch.Generator(device=dev).manual_seed(1234 + rank)
    views_dev = torch.randn(V, 3, 518, 518, device=dev, generator=g)
    coords = synthetic_coords(V, h, w, seed=rank, device=dev)
    n_rows = V * h * w

    def idx_stream(step):
        return np.random.RandomState(1000 * rank + step).randint(0, n_rows, (args.num_iters, 2048))

    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
    seg = []   # ("hp1" | "hp2", start, end) CUDA events recorded on the stream that runs the path

    last_out = {}

    def run_batch(first, n, views, record=False, to_host=False):
        """n images through the public stage-1 call (Stage1Pipeline.run_images): the bank extraction of image i+1 runs
        beside the fit of image i, everything else is ordered by the data dependencies."""
        def finalize(i, out):
            if record:
                last_out.update(out)
            if to_host:
                return out["denoised_feats"].cpu(), out["raw"].cpu()
            return out["denoised_feats"]
        return pipe.run_images(n, lambda i: views, lambda i: coords, lambda i: idx_stream(first + i), finalize,
                               events=seg if record else None, overlap=not args.no_overlap)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(run_step, steps, collate):
        barrier()
        sampler = ClockSampler(local)
        sampler.start()
        l0 = _lib.lib().dvt_launch_count()
        t0, t1 = ev(), ev()
        t0.record()
        outs = run_step(args.warmup, steps)
        if collate and world > 1:  # the single exchange of the path: collate denoised maps for stage 2
            mine = torch.cat([o if torch.is_tensor(o) else o[0].to(dev) for o in outs], 0).contiguous()
            gathered = torch.empty((world,) + tuple(mine.shape), device=dev, dtype=mine.dtype)
            dist.all_gather_into_tensor(gathered, mine)
        t1.record()
        barrier()
        clocks = sampler.stop()
        ms = torch.tensor([t0.elapsed_time(t1)], device=dev)
        if world > 1:
            dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms.item()), clocks, _lib.lib().dvt_launch_count() - l0

    if args.warmup > 0:
        run_batch(0, args.warmup, views_dev)
    ms_total, clocks, launches = timed(lambda first, n: run_batch(first, n, views_dev, record=True), args.steps, collate=True)
    torch.cuda.synchronize()
    if args.dump_outputs and rank == 0:
        os.makedirs(args.dump_outputs, exist_ok=True)
        for name in ("denoised_feats", "raw"):  # 2 x 4.2 MB
            np.save(os.path.join(args.dump_outputs, name + ".npy"), last_out[name].float().cpu().numpy())
    value = world * args.steps / (ms_total / 1000.0)
    # per-path durations INSIDE the timed region (the two paths of neighbouring images overlap, so they do not add up
    # to ms_per_step; each is stretched by the other's share of the SMs / HBM)
    hp1_ms = float(np.mean([a.elapsed_time(b) for k, a, b in seg if k == "hp1"]))
    hp2_ms = float(np.mean([a.elapsed_time(b) for k, a, b in seg if k == "hp2"]))

    e2e = None
    if not args.no_e2e:
        views_host = torch.empty((V, 3, 518, 518), dtype=torch.float32).pin_memory()
        views_host.copy_(views_dev)
        del views_dev
        torch.cuda.empty_cache()
        run_batch(0, 1, views_host, to_host=True)  # warm the staging buffers
        ms_e2e, _, _ = timed(lambda first, n: run_batch(first, n, views_host, to_host=True), args.steps, collate=True)
        h2d = V * 3 * 518 * 518 * 4 + args.num_iters * 2048 * 4
        d2h = 2 * h * w * C * 4
        e2e = {"value": world * args.steps / (ms_e2e / 1000.0), "unit": "images/s", "h2d_bytes_per_step": h2d,
               "d2h_bytes_per_step": d2h, "ms_per_step": ms_e2e / args.steps}
        # The same public call fed with the IMAGE instead of ready-made views (SURVEY.md 8(f-1)): per step one pinned
        # 3.2 MB image goes to the GPU, the 768 random-resized-crop views + their coordinate grids are generated there
        # by dvt_view_crops (crop boxes / flips drawn on the host with the reference's RNG calls), inside the timed region.
        from dvt.dataset import GpuViewGenerator
        del views_host
        gen = GpuViewGenerator((518, 518), num_views=args.views, dtype=torch.float32)
        image_host = torch.randn(3, 518, 518, generator=torch.Generator().manual_seed(rank)).pin_memory()
        views_buf = torch.empty((V, 3, 518, 518), device=dev, dtype=torch.float32)
        coords_of = {}

        def gen_views(i):
            v, c = gen(image_host.to(dev, non_blocking=True), views_out=views_buf)
            coords_of[i] = c
            return v

        def run_from_image(first, n):
            fin = lambda i, out: (out["denoised_feats"].cpu(), out["raw"].cpu())  # noqa: E731
            return pipe.run_images(n, gen_views, lambda i: coords_of[i], lambda i: idx_stream(first + i), fin,
                                   overlap=not args.no_overlap)

        run_from_image(0, 1)
        ms_img, _, _ = timed(run_from_image, args.steps, collate=True)
        e2e["from_image"] = {"value": world * args.steps / (ms_img / 1000.0), "unit": "images/s",
                             "h2d_bytes_per_step": 3 * 518 * 518 * 4 + V * 5 * 4 + args.num_iters * 2048 * 4,
                             "d2h_bytes_per_step": d2h, "ms_per_step": ms_img / args.steps,
                             "note": "views generated on the GPU from one host image per step (dvt_view_crops)"}
        del views_buf

    kr = kernel_rooflines(pipe, args.extract_bsz, dev) if rank == 0 and not args.no_kernel_rooflines else None
    if kr is None and rank == 0:
        kr = {"gemm_ms": None, "gemm_tflops": float("nan"), "gemm_flops": None, "sweep_ms": None, "sweep_gbs": float("nan"),
              "sweep_bytes": None, "sweep_ctas": None, "sweep_full_ms": None, "sweep_full_gbs": float("nan")}

    if rank == 0:
        pk = peaks()
        n_p2 = args.num_iters - 1 - int(0.5 * args.num_iters)
        n_p1 = args.num_iters - n_p2
        # kernel level: the dense Adam sweep and the bf16 GEMM.
        gemm = {"bound": "tensor", "achieved": kr["gemm_tflops"], "peak": pk["bf16_tflops_burst"], "unit": "TFLOP/s",
                    "frac": kr["gemm_tflops"] / pk["bf16_tflops_burst"], "traffic": None,
                    "kernel": "gemm_wgmma_kernel (bf16 wgmma GEMM, the 4 GEMMs of one ViT-B block)",
                    "algorithmic_flops_per_launch_set": kr["gemm_flops"], "ms_per_launch": kr["gemm_ms"],
                    "views_per_launch": args.extract_bsz, "timed": "alone, CUDA events, L2 flushed between launches",
                    "peak_source": pk["source"] + " (bf16 cuBLAS burst: kernel timed alone)"}
        dominant = {"bound": "hbm", "achieved": kr["sweep_gbs"], "peak": pk["hbm_gbs"], "unit": "GB/s",
                    "frac": kr["sweep_gbs"] / pk["hbm_gbs"], "traffic": None,
                    "kernel": "fit_adam_table_kernel (dense Adam sweep of the 19.74 M-parameter hash table), launched as in the "
                              f"timed region: {kr['sweep_ctas']} persistent 1024-thread CTAs (it shares the GPU with the GEMM "
                              "chains of the next two steps, so it is deliberately kept off the other SMs)",
                    "algorithmic_bytes_per_launch": kr["sweep_bytes"], "ms_per_launch": kr["sweep_ms"],
                    "full_grid": {"ms_per_launch": kr["sweep_full_ms"], "achieved": kr["sweep_full_gbs"],
                                  "frac": kr["sweep_full_gbs"] / pk["hbm_gbs"],
                                  "note": "same kernel on 8 x #SM CTAs of 256 threads (the sequential schedule's geometry)"},
                    "timed": "alone, CUDA events around 20 back-to-back launches (474 MB per launch >> L2)",
                    "peak_source": pk["source"] + " (copy bandwidth)"}
        # path level, from the CUDA-event spans INSIDE the timed region (the two paths of neighbouring images overlap,
        # so each span is stretched by the other path's share of the SMs / HBM)
        hp1_tf = V * FLOPS_PER_VIEW / (hp1_ms / 1e3) / 1e12
        hp2_gbs = (n_p1 * FIT_BYTES_P1 + n_p2 * FIT_BYTES_P2) / (hp2_ms / 1e3) / 1e9
        r1 = {"bound": "tensor", "achieved": hp1_tf, "peak": pk["bf16_tflops"], "unit": "TFLOP/s",
              "frac": hp1_tf / pk["bf16_tflops"], "traffic": None, "kernel": "path HP-1: 769 ViT-B/14 forwards (wgmma GEMMs "
              "+ flash attention + LayerNorm)", "ms_per_image": hp1_ms, "peak_source": pk["source"] + " (sustained bf16 cuBLAS)"}
        r2 = {"bound": "hbm", "achieved": hp2_gbs, "peak": pk["hbm_gbs"], "unit": "GB/s", "frac": hp2_gbs / pk["hbm_gbs"],
              "traffic": None, "kernel": "path HP-2: 2000-step neural-field fit (SURVEY 8(d) algorithmic bytes / span)",
              "ms_per_image": hp2_ms, "peak_source": pk["source"] + " (copy bandwidth)"}
        other = [gemm, r1, r2]
        line = {"metric": "images/sec stage-1 denoise (ViT-B/14, 518^2, 2k-iter fit)", "value": value, "unit": "images/s",
                "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_total / args.steps,
                "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16 (ViT) / tf32x3 (fit)",
                "data": "synthetic",
                "config": workload_config(args, world),
                "arm_notes": ("schedule: one image after the other" if args.no_overlap else
                              "schedule: bank extraction of image i+1 overlaps the fit of image i (2 bank buffers)"),
                "clocks": clocks, "gpu_launches": int(launches), "roofline": dominant, "roofline_other": other}
        if e2e is not None:
            line["e2e"] = e2e
        if world == 1 and not args.no_library_bar:
            # BASELINE.md 4.5: the reference's op sequence through the vendor libraries on this same GPU
            sys.path.insert(0, os.path.join(ROOT, "tools"))
            import library_bar
            del pipe
            torch.cuda.empty_cache()
            bar = library_bar.measure(dev, views=V, num_iters=args.num_iters)
            fit_ours_s = hp2_ms / 1e3
            bar["ours"] = {"fit_s_per_image_in_region": fit_ours_s, "hp1_s_per_image_in_region": hp1_ms / 1e3,
                           "images_per_s": value}
            bar["fit_wall_clock_ratio"] = bar["fit_s_per_image"] / fit_ours_s      # north_star target: >= 10
            bar["images_per_s_ratio"] = {k: value / v for k, v in bar["images_per_s"].items()}
            line["library_bar"] = bar
        if world == 1 and not args.no_cpu_baseline:
            line["cpu_baseline"] = cpu_reference_rate(args)
        print(json.dumps(line))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
