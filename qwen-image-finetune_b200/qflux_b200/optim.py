"""Fused clip + AdamW for the LoRA parameters of a fused MMDiT (SURVEY.md §8 f1).

Mirrors what the reference's step body does after `accelerator.backward(loss)`
(/root/reference/src/qflux/trainer/base_trainer.py:528-533): `clip_gradients()` (:449-455, global L2 norm over the trainable
parameters, max_grad_norm) -> `optimizer.step()` (torch.optim.AdamW by default, :884-916 / config.py:534) -> `zero_grad()`.
The gradient is the model's flat fp32 accumulator (all-reduced by the caller for data parallel runs); nothing synchronises
with the host.  Moments are kept in fp32 (torch keeps them in the parameter dtype, bf16) — documented deviation, DESIGN.md.
"""
from __future__ import annotations

import torch

from . import lib


class FusedLoraAdamW(torch.optim.Optimizer):
    """A `torch.optim.Optimizer` over the model's LoRA parameters (so `get_scheduler(...)` / any `LRScheduler` drives `param_groups`
    exactly as with the reference's AdamW), whose `step()` is one fused kernel reading the model's flat fp32 gradient."""

    def __init__(self, model, lr: float = 1e-4, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 1e-2,
                 max_grad_norm: float = 1.0):
        if model.G32 is None:
            raise lib.QfxError("attach a LoRA adapter (model.add_adapter) before building the optimizer")
        super().__init__(list(model.parameters()), dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay))
        self.model = model
        self.max_grad_norm = max_grad_norm
        self.grad_divisor = 1  # how many per-rank / per-micro-step gradients were SUMMED into model.G32 (set by _sync_and_step)
        self.step_count = 0
        n = model.G32.numel()
        self.exp_avg = torch.zeros(n, device=model.dev, dtype=torch.float32)
        self.exp_avg_sq = torch.zeros(n, device=model.dev, dtype=torch.float32)
        self.grad_norm_sq = torch.zeros(1, device=model.dev, dtype=torch.float32)
        self._norm_parts = torch.zeros(lib.DET_NORM_PARTIALS, device=model.dev, dtype=torch.float32)  # deterministic norm
        members = []
        for full, pA, pB, ga, gb, d_in, d_out in model._all_members():
            members += [(pA.data, ga), (pB.data, gb)]
        self._tables = lib.adamw_tables(members, model.dev)

    @torch.no_grad()
    def step(self, closure=None, *, grad_divisor=None):
        """torch.optim contract: the first positional argument is `closure` (accelerate's AcceleratedOptimizer calls `step(closure)`).
        grad = model.G32 / divisor, clipped to max_grad_norm, where the divisor (ranks x accumulated micro-steps, i.e. the SUM in G32 ->
        the mean) is `grad_divisor` if given, else what `_sync_and_step` stored in `self.grad_divisor` after the all-reduce, else 1.
        Returns the closure's loss (None without one); ||grad||^2 stays on the device in `self.grad_norm_sq`."""
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        div = grad_divisor if grad_divisor is not None else self.grad_divisor
        g = self.param_groups[0]
        self.step_count += 1
        args = (self._tables, self.model.G32, self.exp_avg, self.exp_avg_sq, self.grad_norm_sq, 1.0 / float(div), self.max_grad_norm,
                g["lr"], g["betas"][0], g["betas"][1], g["eps"], g["weight_decay"], self.step_count)
        if torch.are_deterministic_algorithms_enabled():  # the clip's norm summed in a fixed order: bit-reproducible
            lib.fused_adamw_det(*args, scratch=self._norm_parts)
        else:
            lib.fused_adamw(*args)
        return loss

    def zero_grad(self, set_to_none: bool = True):
        self.model.G32.zero_()

    def state_dict(self):
        sd = super().state_dict()
        sd["fused"] = dict(step=self.step_count, exp_avg=self.exp_avg, exp_avg_sq=self.exp_avg_sq)
        return sd

    def load_state_dict(self, sd):
        sd = dict(sd)
        fused = sd.pop("fused")
        super().load_state_dict(sd)
        self.step_count = int(fused["step"])
        self.exp_avg.copy_(fused["exp_avg"])
        self.exp_avg_sq.copy_(fused["exp_avg_sq"])
