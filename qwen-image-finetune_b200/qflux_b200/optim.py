"""Fused clip + optimizer step for the LoRA parameters of a fused MMDiT (SURVEY.md §8 f1): AdamW, Prodigy and 8-bit Adam.

Mirrors what the reference's step body does after `accelerator.backward(loss)`
(/root/reference/src/qflux/trainer/base_trainer.py:528-533): `clip_gradients()` (:449-455, global L2 norm over the trainable
parameters, max_grad_norm) -> `optimizer.step()` (torch.optim.AdamW by default, :884-916 / config.py:534; prodigyopt.Prodigy in
four of the shipped configs, bitsandbytes.optim.Adam8bit in eight) -> `zero_grad()`.
The gradient is the model's flat fp32 accumulator (all-reduced by the caller for data parallel runs); nothing synchronises
with the host.  Moments are kept in fp32 (torch keeps them in the parameter dtype, bf16) — documented deviation, DESIGN.md.

With `shard_state=True` (data parallel, world > 1) each rank keeps the optimizer state of its slice of the flat gradient only
(sharding.SlicePlan, ZeRO stage 1): `step()` reduce-scatters the gradient, clips with the norm summed over the slices, steps the slice
and all-gathers the updated LoRA weights (sharding.ShardExchange); `_sync_and_step` then leaves the gradient exchange to it.
"""
from __future__ import annotations

import math

import torch
import torch.distributed as dist

from . import lib


class FusedLoraOptimizer(torch.optim.Optimizer):
    """A `torch.optim.Optimizer` over the model's LoRA parameters (so `get_scheduler(...)` / any `LRScheduler` drives `param_groups`
    exactly as with the reference's optimizer), whose `step()` runs fused kernels reading the model's flat fp32 gradient.
    Subclasses implement `_step(pre_scale)` and, for `shard_state=True`, `_step_slice(pre_scale)`.

    shard_state=True shards the optimizer state across the data-parallel ranks (torch.distributed initialised, world > 1): this rank
    allocates and steps the state of its slice of the flat gradient only, and `step()` runs the exchange itself — reduce-scatter of
    the gradient summed over ranks, the clip's norm summed over the slices in rank order (the same on every run for a given world size,
    not the replicated optimizer's bits), the step of the slice, then the all-gather of the updated LoRA weights.  Every rank must call
    `step()` and `state_dict()` (collectives); `state_dict()` returns the replicated optimizer's format with the whole state gathered,
    and `load_state_dict()` keeps this rank's slice, so checkpoints move between sharded and replicated runs and across world sizes.
    Callers: `train_step` (QwenImageEditStep / FluxKontextStep) and the loop of INTEGRATION.md level 2.  In the reference's own loop
    body (integration.patch_trainer) G32 holds one rank's last micro-step, as for the replicated fused optimizers, so it is not a
    supported caller; patch_trainer never builds a sharded optimizer."""

    def __init__(self, model, defaults: dict, max_grad_norm: float, shard_state: bool = False):
        if model.G32 is None:
            raise lib.QfxError("attach a LoRA adapter (model.add_adapter) before building the optimizer")
        if shard_state:
            if not (dist.is_available() and dist.is_initialized()):
                raise lib.QfxError(f"{type(self).__name__}: shard_state=True needs an initialised torch.distributed process group (the "
                                   "state is split across its data-parallel ranks)")
            if dist.get_world_size() < 2:
                raise lib.QfxError(f"{type(self).__name__}: shard_state=True needs a data-parallel world of 2 or more ranks, got 1")
        super().__init__(list(model.parameters()), defaults)
        self.model = model
        self.max_grad_norm = max_grad_norm
        self.grad_divisor = 1  # how many per-rank / per-micro-step gradients were SUMMED into model.G32 (set by _sync_and_step)
        self.grad_norm_sq = torch.zeros(1, device=model.dev, dtype=torch.float32)
        members = []
        for full, pA, pB, ga, gb, d_in, d_out in model._all_members():
            members += [(pA.data, ga), (pB.data, gb)]
        self._members = members
        self.shard_state = bool(shard_state)
        self._plan = self._exchange = None
        self._lo, self._hi = 0, model.G32.numel()  # the flat-gradient range whose state this rank keeps
        if not self.shard_state:
            self._tables = lib.adamw_tables(members, model.dev)
        else:  # tables in gradient order, so that a slice's chunks are a contiguous range of them
            from .sharding import ShardExchange, SlicePlan
            self._plan = SlicePlan(members, model.G32.numel(), dist.get_world_size())
            self._tables = lib.adamw_tables(self._plan.members, model.dev)
            self._exchange = ShardExchange(model, self._plan, self._tables)
            self._rank = dist.get_rank()
            self._lo, self._hi = self._plan.bounds[self._rank]
            self._chunk_range = self._plan.chunk_ranges[self._rank]
            self._norm_part = torch.zeros(1, device=model.dev, dtype=torch.float32)  # this slice's ||grad * pre_scale||^2
            self._norm_scratch = torch.zeros(lib.DET_NORM_PARTIALS, device=model.dev, dtype=torch.float32)

    @property
    def _n_state(self):
        return self._hi - self._lo

    def _gather(self, x):
        """The whole of a state array kept per slice of the flat gradient (replicated: x itself)."""
        return x if self._plan is None else self._exchange.gather_ranges(x, self._plan.bounds)

    def _mine(self, full):
        """This rank's part of a whole state array of the flat-gradient layout."""
        return full[self._lo: self._hi]

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
        if self._plan is None:
            self._step(1.0 / float(div))
        else:
            self._sharded_step(1.0 / float(div))
        return loss

    def _sharded_step(self, pre_scale):
        if not self._ready_to_step():
            return
        ex = self._exchange
        ex.reduce_scatter()
        g32 = self.model.G32  # the deterministic exchange may have moved it into peer memory
        lib.sumsq_det(g32[self._lo: self._hi], pre_scale, self._norm_part, scratch=self._norm_scratch)
        ex.gather_sum(self._norm_part, self.grad_norm_sq)
        self._step_slice(pre_scale)
        ex.gather_weights()

    def _ready_to_step(self):
        """False when this step changes nothing on any rank (Prodigy at lr == 0): the exchange is skipped too."""
        return True

    def zero_grad(self, set_to_none: bool = True):
        self.model.G32.zero_()


class FusedLoraAdamW(FusedLoraOptimizer):
    """torch.optim.AdamW after the clip, as one fused kernel (plus the norm)."""

    def __init__(self, model, lr: float = 1e-4, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 1e-2,
                 max_grad_norm: float = 1.0, shard_state: bool = False):
        super().__init__(model, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay), max_grad_norm, shard_state)
        self.step_count = 0
        n = self._n_state
        self.exp_avg = torch.zeros(n, device=model.dev, dtype=torch.float32)
        self.exp_avg_sq = torch.zeros(n, device=model.dev, dtype=torch.float32)
        self._norm_parts = torch.zeros(lib.DET_NORM_PARTIALS, device=model.dev, dtype=torch.float32)  # deterministic norm

    def _step(self, pre_scale):
        g = self.param_groups[0]
        self.step_count += 1
        args = (self._tables, self.model.G32, self.exp_avg, self.exp_avg_sq, self.grad_norm_sq, pre_scale, self.max_grad_norm,
                g["lr"], g["betas"][0], g["betas"][1], g["eps"], g["weight_decay"], self.step_count)
        if torch.are_deterministic_algorithms_enabled():  # the clip's norm summed in a fixed order: bit-reproducible
            lib.fused_adamw_det(*args, scratch=self._norm_parts)
        else:
            lib.fused_adamw(*args)

    def _step_slice(self, pre_scale):
        g = self.param_groups[0]
        self.step_count += 1
        lib.fused_adamw_slice(self._tables, self._chunk_range, self._lo, self.model.G32, self.exp_avg, self.exp_avg_sq, self.grad_norm_sq,
                              pre_scale, self.max_grad_norm, g["lr"], g["betas"][0], g["betas"][1], g["eps"], g["weight_decay"],
                              self.step_count)

    def state_dict(self):
        sd = super().state_dict()
        sd["fused"] = dict(step=self.step_count, exp_avg=self._gather(self.exp_avg), exp_avg_sq=self._gather(self.exp_avg_sq))
        return sd

    def load_state_dict(self, sd):
        sd = dict(sd)
        fused = sd.pop("fused")
        super().load_state_dict(sd)
        self.step_count = int(fused["step"])
        self.exp_avg.copy_(self._mine(fused["exp_avg"]))
        self.exp_avg_sq.copy_(self._mine(fused["exp_avg_sq"]))


class FusedLoraAdam8bit(FusedLoraOptimizer):
    """bitsandbytes' `optim.Adam8bit` (block-wise 8-bit Adam) after the clip, as fused kernels over the flat gradient (qfx.h
    qfx_fused_adam8bit): the constructor takes Adam8bit's arguments and defaults, plus `max_grad_norm`.  `optim_bits` is ignored
    (Adam8bit always keeps 8-bit states) and so is `is_paged` (paging only decides where the state memory lives); `amsgrad`,
    `percentile_clipping != 100`, `block_wise=False` and `args` are refused.  A step with lr == 0 still updates the states and the step
    count, as in bitsandbytes.

    State, per LoRA tensor in member order (A then B of each adapted Linear), laid out as bitsandbytes' per-parameter
    `state1 / state2 / absmax1 / absmax2 / qmap1 / qmap2` concatenated:
      * numel >= min_8bit_size: uint8 codes `state1[off: off + numel]`, `state2[...]` (off = the tensor's offset in the flat gradient,
        row-major over the tensor) and fp32 `absmax1[a: a + ceil(numel / 256)]`, `absmax2[...]` (a = `state_offsets[i]`);
      * smaller tensors: fp32 `s1_32[a: a + numel]`, `s2_32[...]`; their code bytes stay 0;
      * `qmap1` / `qmap2`: the signed / unsigned dynamic maps, shared by every tensor (bitsandbytes keeps one copy per tensor).
    `state_dict()` carries all of it and the step count."""

    def __init__(self, model, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0, amsgrad: bool = False,
                 optim_bits: int = 32, args=None, min_8bit_size: int = 4096, percentile_clipping: int = 100, block_wise: bool = True,
                 is_paged: bool = False, max_grad_norm: float = 1.0, shard_state: bool = False):
        if amsgrad:
            raise lib.QfxError("FusedLoraAdam8bit: amsgrad=True is not implemented")
        if percentile_clipping != 100:
            raise lib.QfxError(f"FusedLoraAdam8bit: percentile_clipping={percentile_clipping} is not implemented (it needs a 100-step "
                               "history of gradient norms)")
        if not block_wise:
            raise lib.QfxError("FusedLoraAdam8bit: block_wise=False is not implemented (only block-wise 8-bit states)")
        if args is not None:
            raise lib.QfxError("FusedLoraAdam8bit: args (a bitsandbytes optimizer config object) is not supported; pass the arguments "
                               "themselves")
        super().__init__(model, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay), max_grad_norm, shard_state)
        self.min_8bit_size = int(min_8bit_size)
        n, dev = self._n_state, model.dev
        offsets, n_absmax, n_small = lib.adam8bit_layout(self._members, self.min_8bit_size)
        if self._plan is not None:
            # absmax blocks and fp32 states laid out in the plan's member order, where each slice's are a contiguous range; the
            # state_dict keeps the replicated layout (`_perm`: position in it of each element of the plan's layout)
            full = offsets
            offsets, n_absmax, n_small = lib.adam8bit_layout(self._plan.members, self.min_8bit_size)
            self._perm = {"absmax": torch.zeros(n_absmax, dtype=torch.int64), "s": torch.zeros(n_small, dtype=torch.int64)}
            for j, (p, _) in enumerate(self._plan.members):
                k, c = ("absmax", -(-p.numel() // lib.ADAM8BIT_BLOCK)) if p.numel() >= self.min_8bit_size else ("s", p.numel())
                o = full[self._plan.order[j]]
                self._perm[k][offsets[j]: offsets[j] + c] = torch.arange(o, o + c)
            self._perm = {k: v.to(dev) for k, v in self._perm.items()}
            self._absmax_ranges, self._small_ranges = self._state_ranges(offsets, n_absmax, n_small)
            a0, s0 = self._absmax_ranges[self._rank][0], self._small_ranges[self._rank][0]
            offsets = [o - (a0 if p.numel() >= self.min_8bit_size else s0) for (p, _), o in zip(self._plan.members, offsets)]
            n_absmax = self._absmax_ranges[self._rank][1] - a0
            n_small = self._small_ranges[self._rank][1] - s0
        self.state_offsets = torch.tensor(offsets, dtype=torch.int64).to(dev)
        self.state1 = torch.zeros(n, device=dev, dtype=torch.uint8)
        self.state2 = torch.zeros(n, device=dev, dtype=torch.uint8)
        self.absmax1 = torch.zeros(max(1, n_absmax), device=dev, dtype=torch.float32)  # one element when nothing is 8-bit: the C side
        self.absmax2 = torch.zeros(max(1, n_absmax), device=dev, dtype=torch.float32)  # takes no null pointers
        self.s1_32 = torch.zeros(max(1, n_small), device=dev, dtype=torch.float32)
        self.s2_32 = torch.zeros(max(1, n_small), device=dev, dtype=torch.float32)
        self.qmap1 = lib.dynamic_map(signed=True).to(dev)
        self.qmap2 = lib.dynamic_map(signed=False).to(dev)
        self.step_count = 0
        self._norm_parts = torch.zeros(lib.DET_NORM_PARTIALS, device=dev, dtype=torch.float32)

    _STATE = ("state1", "state2", "absmax1", "absmax2", "s1_32", "s2_32", "qmap1", "qmap2")

    def _state_ranges(self, offsets, n_absmax, n_small):
        """Per rank: the [start, end) of its slice's absmax blocks and of its fp32 small-tensor states in the whole arrays."""
        absmax, small = [], []
        for q in range(self._plan.world):
            a, s = [], []
            for i, e0, e1 in self._plan.pieces(q):
                if self._plan.members[i][0].numel() >= self.min_8bit_size:
                    a += [offsets[i] + e0 // lib.ADAM8BIT_BLOCK, offsets[i] + -(-e1 // lib.ADAM8BIT_BLOCK)]
                else:
                    s += [offsets[i] + e0, offsets[i] + e1]
            absmax.append((min(a), max(a)) if a else None)
            small.append((min(s), max(s)) if s else None)
        for ranges, total in ((absmax, n_absmax), (small, n_small)):  # an empty range sits where the next one starts
            nxt = total
            for q in reversed(range(len(ranges))):
                ranges[q] = ranges[q] or (nxt, nxt)
                nxt = ranges[q][0]
        return absmax, small

    def _whole(self, k):
        x = getattr(self, k)
        if self._plan is None or k.startswith("qmap"):
            return x
        if k.startswith("state"):
            return self._gather(x)
        ranges = self._absmax_ranges if k.startswith("absmax") else self._small_ranges
        mine = self._exchange.gather_ranges(x[: ranges[self._rank][1] - ranges[self._rank][0]], ranges)
        whole = torch.empty_like(mine).index_copy_(0, self._perm["absmax" if k.startswith("absmax") else "s"], mine)
        return whole if whole.numel() else x.new_zeros(1)

    def _part(self, k, full):
        if self._plan is None or k.startswith("qmap"):
            return full
        if k.startswith("state"):
            return self._mine(full)
        a, b = (self._absmax_ranges if k.startswith("absmax") else self._small_ranges)[self._rank]
        perm = self._perm["absmax" if k.startswith("absmax") else "s"]
        return full.to(perm.device)[perm[a:b]]

    def _step(self, pre_scale):
        g = self.param_groups[0]
        self.step_count += 1
        lib.fused_adam8bit(self._tables, self.state_offsets, self.model.G32, self.state1, self.state2, self.absmax1, self.absmax2,
                           self.s1_32, self.s2_32, self.qmap1, self.qmap2, self.grad_norm_sq, self._norm_parts, pre_scale,
                           self.max_grad_norm, g["lr"], g["betas"][0], g["betas"][1], g["eps"], g["weight_decay"], self.step_count,
                           self.min_8bit_size)

    def _step_slice(self, pre_scale):
        g = self.param_groups[0]
        self.step_count += 1
        lib.fused_adam8bit_slice(self._tables, self._chunk_range, self._lo, self.state_offsets, self.model.G32, self.state1, self.state2,
                                 self.absmax1, self.absmax2, self.s1_32, self.s2_32, self.qmap1, self.qmap2, self.grad_norm_sq, pre_scale,
                                 self.max_grad_norm, g["lr"], g["betas"][0], g["betas"][1], g["eps"], g["weight_decay"], self.step_count,
                                 self.min_8bit_size)

    def state_dict(self):
        sd = super().state_dict()
        sd["fused"] = dict(step=self.step_count, **{k: self._whole(k) for k in self._STATE})
        return sd

    def load_state_dict(self, sd):
        sd = dict(sd)
        fused = sd.pop("fused")
        super().load_state_dict(sd)
        self.step_count = int(fused["step"])
        for k in self._STATE:
            part = self._part(k, fused[k])
            getattr(self, k)[: part.numel()].copy_(part)


class FusedLoraProdigy(FusedLoraOptimizer):
    """prodigyopt.Prodigy (Mishchenko & Defazio, "Prodigy: An Expeditiously Adaptive Parameter-Free Learner") after the clip, as fused
    kernels over the flat gradient (qfx.h qfx_fused_prodigy): the constructor takes prodigyopt's arguments and defaults, plus
    `max_grad_norm`.  prodigyopt reads its two global sums back with `.item()` for every parameter tensor; here they stay on the
    device, and so do d, d_max, d_numerator and k (`self.scalars`, fp64; `self.d` is d as a device tensor).  A step with lr == 0
    (the first step of a warm-up schedule) changes nothing, as in prodigyopt, and launches nothing.  p0 is the parameters at the first
    `step()` call.  m, v, s are fp32 and p0 bf16 (prodigyopt keeps all four in the parameter dtype); `slice_p != 1` and FSDP are
    refused."""

    def __init__(self, model, lr: float = 1.0, betas=(0.9, 0.999), beta3=None, eps: float = 1e-8, weight_decay: float = 0.0,
                 decouple: bool = True, use_bias_correction: bool = False, safeguard_warmup: bool = False, d0: float = 1e-6,
                 d_coef: float = 1.0, growth_rate: float = float("inf"), fsdp_in_use: bool = False, slice_p: int = 1,
                 max_grad_norm: float = 1.0, shard_state: bool = False):
        if slice_p != 1:
            raise lib.QfxError(f"FusedLoraProdigy: slice_p={slice_p} is not implemented (the kernels estimate d from every element)")
        if fsdp_in_use:
            raise lib.QfxError("FusedLoraProdigy: fsdp_in_use=True is not implemented (data-parallel ranks hold the all-reduced gradient "
                               "and the same parameters, so they compute the same d without it)")
        if not d0 > 0:
            raise lib.QfxError(f"FusedLoraProdigy: d0 must be > 0, got {d0}")
        super().__init__(model, dict(lr=lr, betas=tuple(betas), beta3=beta3, eps=eps, weight_decay=weight_decay, decouple=decouple,
                                     use_bias_correction=use_bias_correction, safeguard_warmup=safeguard_warmup, d0=d0, d_coef=d_coef,
                                     growth_rate=growth_rate), max_grad_norm, shard_state)
        n, dev = self._n_state, model.dev
        self.exp_avg = torch.zeros(n, device=dev, dtype=torch.float32)
        self.exp_avg_sq = torch.zeros(n, device=dev, dtype=torch.float32)
        self.s = torch.zeros(n, device=dev, dtype=torch.float32)
        self.p0 = torch.zeros(n, device=dev, dtype=torch.bfloat16)
        self.p0_set = False
        self.scalars = torch.zeros(lib.PRODIGY_SCALARS, device=dev, dtype=torch.float64)
        self.scalars[lib.PRODIGY_D] = self.scalars[lib.PRODIGY_D_MAX] = d0
        self._scratch = torch.zeros(lib.prodigy_scratch_floats(self._tables), device=dev, dtype=torch.float32)
        if self._plan is not None:  # every chunk's (sum g (p0 - p), sum |s|): this rank's written by pass A, the others gathered,
            n_chunks = len(self._plan.chunks)  # then put in the replicated tables' chunk order, which the scalar update sums in
            self._part = torch.zeros(n_chunks, 2, device=dev, dtype=torch.float64)
            self._part_table = torch.zeros(n_chunks, 2, device=dev, dtype=torch.float64)
            self._table_chunk = torch.tensor(self._plan.table_chunk, dtype=torch.int64).to(dev)

    @property
    def d(self):
        """Prodigy's current step-size estimate d (0-dim fp64 device tensor; reading it as a number synchronises)."""
        return self.scalars[lib.PRODIGY_D]

    @property
    def d_max(self):
        return self.scalars[lib.PRODIGY_D_MAX]

    @property
    def k(self):
        """Steps that updated d and the parameters (prodigyopt's group['k'])."""
        return self.scalars[lib.PRODIGY_K]

    def _capture_p0(self):
        if self._plan is not None:
            lib.lora_pack(self._tables, self._chunk_range, self._lo, self._hi, self.p0)
        else:
            for p, off in self._members:
                self.p0[off: off + p.numel()].view(p.shape).copy_(p)
        self.p0_set = True

    def _ready_to_step(self):
        if not self.p0_set:
            self._capture_p0()
        return self.param_groups[0]["lr"] != 0

    def _step_slice(self, pre_scale):
        g = self.param_groups[0]
        beta1, beta2 = g["betas"]
        beta3 = g["beta3"] if g["beta3"] is not None else math.sqrt(beta2)
        lib.prodigy_slice_partials(self._tables, self._chunk_range, self._lo, self.model.G32, self.exp_avg, self.exp_avg_sq, self.s,
                                   self.p0, self.scalars, self.grad_norm_sq, self._part, pre_scale, self.max_grad_norm, g["lr"], beta1,
                                   beta2, beta3, g["weight_decay"], g["decouple"], g["use_bias_correction"], g["safeguard_warmup"],
                                   g["d0"])
        self._exchange.gather_rows(self._part)
        self._part_table.index_copy_(0, self._table_chunk, self._part)
        lib.prodigy_slice_update(self._tables, self._chunk_range, self._lo, self.model.G32.numel(), self.exp_avg, self.exp_avg_sq,
                                 self.scalars, self._part_table, g["lr"], beta1, beta2, beta3, g["eps"], g["weight_decay"], g["decouple"],
                                 g["use_bias_correction"], g["d0"], g["d_coef"], g["growth_rate"])

    def _step(self, pre_scale):
        g = self.param_groups[0]
        if not self.p0_set:
            self._capture_p0()
        if g["lr"] == 0:
            return
        beta1, beta2 = g["betas"]
        beta3 = g["beta3"] if g["beta3"] is not None else math.sqrt(beta2)
        lib.fused_prodigy(self._tables, self.model.G32, self.exp_avg, self.exp_avg_sq, self.s, self.p0, self.scalars, self.grad_norm_sq,
                          self._scratch, pre_scale, self.max_grad_norm, g["lr"], beta1, beta2, beta3, g["eps"], g["weight_decay"],
                          g["decouple"], g["use_bias_correction"], g["safeguard_warmup"], g["d0"], g["d_coef"], g["growth_rate"])

    def state_dict(self):
        sd = super().state_dict()
        sd["fused"] = dict(exp_avg=self._gather(self.exp_avg), exp_avg_sq=self._gather(self.exp_avg_sq), s=self._gather(self.s),
                           p0=self._gather(self.p0), p0_set=self.p0_set, scalars=self.scalars)
        return sd

    def load_state_dict(self, sd):
        sd = dict(sd)
        fused = sd.pop("fused")
        super().load_state_dict(sd)
        for k in ("exp_avg", "exp_avg_sq", "s", "p0"):
            getattr(self, k).copy_(self._mine(fused[k]))
        self.scalars.copy_(fused["scalars"])
        self.p0_set = bool(fused["p0_set"])
