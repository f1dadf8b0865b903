"""`FusedAdamW`: torch.optim.AdamW semantics (reference main_denoiser.py:176-180: betas (0.9, 0.999), eps 1e-8, decoupled
weight decay on every parameter, one parameter group) as ONE kernel launch per step.

All parameters live in one flat fp32 buffer (the module's Parameters become views of it), and so do their gradients and
both moments: `zero_grad` is one memset, the data-parallel gradient exchange is ONE all-reduce of the flat gradient
(32.6 MB for the ViT-B denoiser; the reference wraps the model in DistributedDataParallel, main_denoiser.py:139) and the
update is `dvt_adamw` over the flat buffers.  `state_dict()` / `load_state_dict()` use torch.optim's layout (per-parameter
`step` / `exp_avg` / `exp_avg_sq`, `param_groups`), so checkpoints interchange with the reference's
(`{"denoiser", "optimizer", "step"}`, main_denoiser.py:248-252)."""
from __future__ import annotations

from typing import Dict, Iterable, List

import torch

from . import train_ops


class FusedAdamW:
    def __init__(self, params: Iterable[torch.nn.Parameter], lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8,
                 weight_decay: float = 1e-2):
        self.params: List[torch.nn.Parameter] = [p for p in params if p.requires_grad]
        assert self.params, "FusedAdamW: no trainable parameters"
        dev = self.params[0].device
        if dev.type != "cuda":
            raise RuntimeError("FusedAdamW needs CUDA parameters (no CPU fallback)")
        self.offsets, total = [], 0
        for p in self.params:
            assert p.device == dev and p.dtype == torch.float32
            self.offsets.append(total)
            total += (p.numel() + 3) // 4 * 4          # every tensor starts on a 16-byte boundary
        self.numel = total
        self.flat_p = torch.zeros(total, device=dev, dtype=torch.float32)
        self.flat_g = torch.zeros_like(self.flat_p)
        self.exp_avg = torch.zeros_like(self.flat_p)
        self.exp_avg_sq = torch.zeros_like(self.flat_p)
        for p, off in zip(self.params, self.offsets):
            view = self.flat_p[off:off + p.numel()].view_as(p)
            view.copy_(p.data)
            p.data = view
            p.grad = self.flat_g[off:off + p.numel()].view_as(p)
        self.param_groups = [{"lr": lr, "betas": tuple(betas), "eps": eps, "weight_decay": weight_decay, "amsgrad": False,
                              "maximize": False, "foreach": None, "capturable": False, "differentiable": False,
                              "fused": True, "params": list(range(len(self.params)))}]
        self.step_count = 0

    # ---- torch.optim.Optimizer surface -------------------------------------------------------------------------------
    def zero_grad(self, set_to_none: bool = False):
        self.flat_g.zero_()
        for p, off in zip(self.params, self.offsets):   # autograd may have replaced a .grad (it does not, but stay safe)
            if p.grad is None or p.grad.data_ptr() != self.flat_g.data_ptr() + 4 * off:
                p.grad = self.flat_g[off:off + p.numel()].view_as(p)

    def sync_grads(self, world_size: int = 1):
        """Data-parallel gradient average: ONE all-reduce over NVLink of the flat gradient buffer."""
        if world_size > 1:
            import torch.distributed as dist
            dist.all_reduce(self.flat_g, op=dist.ReduceOp.SUM)
            self.flat_g.div_(world_size)

    @torch.no_grad()
    def step(self):
        g = self.param_groups[0]
        self.step_count += 1
        train_ops.adamw_(self.flat_p, self.flat_g, self.exp_avg, self.exp_avg_sq, lr=g["lr"], betas=g["betas"], eps=g["eps"],
                         weight_decay=g["weight_decay"], step=self.step_count)
        # the kernel writes the flat buffer behind autograd's back: bump the parameters' version counters so that caches keyed
        # on them (the bf16 weight copies of dvt.models) see the update
        torch.autograd.graph.increment_version(self.params)

    def state_dict(self) -> Dict:
        state = {}
        for i, (p, off) in enumerate(zip(self.params, self.offsets)):
            sl = slice(off, off + p.numel())
            state[i] = {"step": torch.tensor(float(self.step_count)), "exp_avg": self.exp_avg[sl].view_as(p).clone(),
                        "exp_avg_sq": self.exp_avg_sq[sl].view_as(p).clone()}
        return {"state": state if self.step_count > 0 else {}, "param_groups": [dict(g) for g in self.param_groups]}

    def load_state_dict(self, sd: Dict):
        for k, v in sd["param_groups"][0].items():
            if k != "params":
                self.param_groups[0][k] = v
        for i, st in sd.get("state", {}).items():
            i = int(i)
            p, off = self.params[i], self.offsets[i]
            sl = slice(off, off + p.numel())
            self.exp_avg[sl].copy_(st["exp_avg"].reshape(-1))
            self.exp_avg_sq[sl].copy_(st["exp_avg_sq"].reshape(-1))
            self.step_count = int(float(st["step"]))
