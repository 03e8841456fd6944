"""Training-step recipes on top of the fused model — mirrors of the reference trainers' `_compute_loss`.

  QwenImageEditStep.compute_loss   <- /root/reference/src/qflux/trainer/qwen_image_edit_trainer.py:777-849 (+ _get_sigmas :851-861)
  loss kinds                       <- /root/reference/src/qflux/losses/{mse_loss,edit_mask_loss,attention_mask_loss}.py
  gradient sync / clip             <- /root/reference/src/qflux/trainer/base_trainer.py:383-388 (DDP over the LoRA params), :449-455

Differences that are deliberate (SURVEY.md §5 caveat, DESIGN.md):
  * the per-step `deepcopy(scheduler)` + `.nonzero().item()` host syncs are gone: sigma = (1000 - idx)/1000 is computed on
    the host from the CPU uniform draw (same RNG stream as the reference) and uploaded asynchronously;
  * LoRA gradients are mean-all-reduced explicitly every optimizer step (one NCCL all-reduce over one flat fp32 buffer).
"""
from __future__ import annotations

import torch
import torch.distributed as dist

from . import lib
from .mmdit_base import GraphCache
from .qwen_model import BF, QwenImageB200


def token_weights_and_norm(kind, B, L, C, weighting=None, attention_mask=None, edit_mask=None, fg=2.0, bg=1.0, eps=1e-12):
    """(w [B, L] fp32 on host or device, norm) with  loss = norm * sum w * (pred - target)^2  for reduction='mean'.
    kind: "mse" (MseLoss), "mask_edit" (MaskEditLoss), "attention_mask" (AttentionMaskMseLoss)."""
    dev = None
    for t in (weighting, attention_mask, edit_mask):
        if t is not None:
            dev = t.device
    w = torch.ones(B, L, dtype=torch.float32, device=dev)
    if weighting is not None:
        w = w * weighting.float().reshape(B, -1)[:, :1]
    if kind == "mse":
        return w, 1.0 / (B * L * C)
    if kind == "mask_edit":
        w = w * ((edit_mask.float() * fg + (1 - edit_mask.float()) * bg) if edit_mask is not None else fg)
        return w, 1.0 / (B * L * C)
    if kind == "attention_mask":
        if edit_mask is not None:
            w = w * (edit_mask.float() * fg + (1 - edit_mask.float()) * bg)
        if attention_mask is None:
            return w, 1.0 / (C * (B * L + eps))
        w = w * attention_mask.float()
        return w, None  # norm needs the valid-token count: computed on device by the caller
    raise ValueError(f"unknown loss kind {kind!r}")


class _FusedStep:
    """What the step recipes share: loss weights, the fused loss + backward tail of `_run`, the autograd entry (`compute_loss`) and
    the fast path (`train_step`) with gradient accumulation (`accelerator.accumulate(...)` around training_step,
    base_trainer.py:518-533, train.gradient_accumulation_steps): micro-steps add into the same flat fp32 LoRA gradient; the exchange +
    clip + optimizer step run on the last one with the mean over micro-steps and ranks (accelerate divides the loss by the number of
    accumulation steps).

    The fused step is ~1,300 (Qwen) to ~3,400 (FLUX with the YAML target set) kernel launches issued from Python through ctypes:
    170-210 ms of host time per step, close to (FLUX: above) the device time.  All of it is shape-static, so `train_step` runs it
    through a CUDA-graph cache (mmdit_base.GraphCache) keyed on the input signature and on whether the micro-step accumulates; every
    replayed step is a handful of small copies plus one graph launch.  The exchange + clip + optimizer stay outside (NCCL, and the
    optimizer's step count is a kernel argument)."""

    def __init__(self, dit, loss_kind: str = "mse", fg: float = 2.0, bg: float = 1.0, max_grad_norm: float = 1.0,
                 gradient_accumulation_steps: int = 1, use_cuda_graph: bool = True):
        self.dit, self.loss_kind, self.fg, self.bg, self.max_grad_norm = dit, loss_kind, fg, bg, max_grad_norm
        self._ones = {}
        self._accumulating = False
        self.gradient_accumulation_steps, self._micro = max(1, int(gradient_accumulation_steps)), 0
        self.use_cuda_graph, self._graphs = bool(use_cuda_graph), GraphCache(16, "the fused step")

    def _dense_loss_weights(self, B, L, C, edit_mask):
        """(w [B, L] fp32 on the device, norm) of a batch whose samples share one resolution."""
        dev = self.dit.dev
        if self.loss_kind == "mse" and edit_mask is None:
            if (B, L) not in self._ones:
                self._ones[(B, L)] = torch.ones(B, L, device=dev)
            return self._ones[(B, L)], 1.0 / (B * L * C)
        w, norm = token_weights_and_norm(self.loss_kind, B, L, C, None, None, None if edit_mask is None else edit_mask.to(dev),
                                         self.fg, self.bg)
        return w.to(dev).contiguous(), norm

    def _var_lengths(self, shapes, L):
        """Pad-to-max multi-resolution batch: img_shapes holds one list of latent (frame, h, w) per sample, target first, then the
        controls.  Returns (target tokens lt, control tokens lc (host lists), padded length Ltot, Lt, Lc (int32 [B] on the device),
        target-token mask [B, L] (host fp32))."""
        dev = self.dit.dev
        lt = [f * h * w for f, h, w in (sh[0] for sh in shapes)]
        lc = [sum(f * h * w for f, h, w in sh[1:]) for sh in shapes]
        Lt = torch.tensor(lt, dtype=torch.int32).to(dev, non_blocking=True)
        Lc = torch.tensor(lc, dtype=torch.int32).to(dev, non_blocking=True)
        amask = (torch.arange(L)[None, :] < torch.tensor(lt)[:, None]).float()
        return lt, lc, max(a + b for a, b in zip(lt, lc)), Lt, Lc, amask

    def _loss_and_backward(self, pred, x0, noise, w, norm):
        """Tail of `_run`: flow-matching loss and its gradient, then the fused backward into the flat LoRA gradient (zeroed first unless
        this micro-step accumulates).  Returns the loss (a workspace scalar)."""
        m = self.dit
        ws = m._ws
        lib.flow_loss(pred, x0, noise, w, norm, ws["loss"], ws["dpred"])
        if not self._accumulating:
            m.G32.zero_()
        m._backward_impl(ws["dpred"])
        return ws["loss"]

    def _autograd_loss(self, args):
        return _StepFn.apply(self, args, *self.dit._lora_params.values())

    def _fused_micro_step(self, args, optimizer):
        self._accumulating = self._micro > 0  # read by _run: keep the gradient of the earlier micro-steps
        loss = self._graphs.run(self.dit, self._run, args, tag=self._accumulating, enabled=self.use_cuda_graph)
        loss = loss.clone()  # the workspace scalar is overwritten by the next step
        self._accumulating = False
        self._micro += 1
        if self._micro >= self.gradient_accumulation_steps:
            _sync_and_step(self.dit, optimizer, self.max_grad_norm, self._micro)
            self._micro = 0
        return loss


def _sync_and_step(dit, optimizer, max_grad_norm, micro_steps: int = 1):
    """Data-parallel tail of a step (base_trainer.py:383-388, 449-455, 528-533): ONE all-reduce(sum) of the flat fp32 LoRA
    gradient, then either the fused clip + AdamW kernel (FusedLoraAdamW reads the accumulator directly) or, for any torch
    optimizer, mean + clip + cast into the bf16 `.grad` views followed by `optimizer.step()`."""
    from .optim import FusedLoraAdamW
    world = 1
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        world = dist.get_world_size()
        dist.all_reduce(dit.G32)
    inner = getattr(optimizer, "optimizer", optimizer)  # accelerate hands the trainer an AcceleratedOptimizer wrapper (.optimizer)
    if isinstance(inner, FusedLoraAdamW):
        inner.max_grad_norm = max_grad_norm
        inner.grad_divisor = world * micro_steps  # G32 holds the SUM over ranks and micro-steps
        optimizer.step()                          # through the wrapper when there is one (step(closure=None) contract)
        return
    dit.finalize_grads(world * micro_steps, max_grad_norm)
    if optimizer is not None:
        optimizer.step()


class _StepFn(torch.autograd.Function):
    """loss = fused(forward -> flow loss -> backward); autograd backward only scales the already computed gradients."""

    @staticmethod
    def forward(ctx, step, args, *params):
        loss = step._run(*args)
        ctx.step = step
        ctx.gen = step.dit._fwd_gen
        return loss.clone().reshape(())

    @staticmethod
    def backward(ctx, g):
        m = ctx.step.dit
        if ctx.gen != m._fwd_gen:
            raise RuntimeError("qflux_b200: backward() of a loss whose fused gradients were overwritten by a later forward of the same model")
        views = m.lora_grad_views((m.G32 * g).to(BF))
        grads = tuple(views[k] for k in m._lora_params)
        return (None, None) + grads


class QwenImageEditStep(_FusedStep):
    def __init__(self, dit: QwenImageB200, loss_kind: str = "mse", fg: float = 2.0, bg: float = 1.0,
                 num_train_timesteps: int = 1000, max_grad_norm: float = 1.0, gradient_accumulation_steps: int = 1,
                 use_cuda_graph: bool = True):
        super().__init__(dit, loss_kind, fg, bg, max_grad_norm, gradient_accumulation_steps, use_cuda_graph)
        self.num_train_timesteps = num_train_timesteps

    # --------------------------------------------------------------------------------------------- internals
    def _sigmas(self, B, u=None):
        if u is None:
            u = torch.rand(B)  # compute_density_for_timestep_sampling("none"): global CPU RNG, like the reference
        idx = (u * self.num_train_timesteps).long()
        timesteps = (self.num_train_timesteps - idx).float()  # scheduler.timesteps = linspace(1, 1000, 1000)[::-1]
        return (timesteps / self.num_train_timesteps)

    def _run(self, image_latents, control_latents, prompt_embeds, img_shapes, noise, sigma, w, norm, var=None):
        m = self.dit
        B, L, C = image_latents.shape
        if var is None:
            packed = torch.empty(B, L + control_latents.shape[1], C, device=m.dev, dtype=BF)
            lib.flow_noisy_input(image_latents, noise, control_latents, sigma, packed)
            pred = m._forward_impl(packed, prompt_embeds, sigma, img_shapes, train=True)
        else:  # multi-resolution pad-to-max batch: per-sample [target | control] concatenation, masks and RoPE
            Lt, Lc, Ltot, txt_len = var
            packed = torch.empty(B, Ltot, C, device=m.dev, dtype=BF)
            lib.flow_noisy_input_var(image_latents, noise, control_latents, sigma, Lt, Lc, packed)
            pred = m._forward_impl(packed, prompt_embeds, sigma, img_shapes, txt_len, train=True)
        return self._loss_and_backward(pred, image_latents, noise, w, norm)

    def _prepare(self, embeddings, noise, u):
        m = self.dit
        dev = m.dev
        x0 = embeddings["image_latents"].to(dev, BF, non_blocking=True).contiguous()
        ctrl = embeddings["control_latents"].to(dev, BF, non_blocking=True).contiguous()
        pe = embeddings["prompt_embeds"].to(dev, BF, non_blocking=True).contiguous()
        B, L, C = x0.shape
        if noise is None:  # like the FLUX trainer (flux_kontext_trainer.py:515-522) the batch may carry its own noise / draw
            noise = embeddings["noise"] if "noise" in embeddings else torch.randn(x0.shape, device=dev, dtype=BF)
        if u is None and "u" in embeddings:
            u = embeddings["u"]
        sigma = self._sigmas(B, u).to(dev, non_blocking=True)
        edit_mask = embeddings.get("edit_mask")
        shapes = embeddings["img_shapes"]
        multi = isinstance(shapes[0][0], (list, tuple)) and any(list(map(tuple, sh)) != list(map(tuple, shapes[0])) for sh in shapes)
        if multi:
            # pad-to-max multi-resolution batch (SURVEY.md §8a a4/a11): token counts come from the latent-space shapes (host
            # metadata), the loss is AttentionMaskMseLoss over the valid target tokens (attention_mask_loss.py:146-226)
            lt, lc, Ltot, Lt, Lc, amask = self._var_lengths(shapes, L)
            mask = embeddings.get("prompt_embeds_mask")
            txt_len = None if mask is None else mask.to(dev).sum(dim=1).to(torch.int32)
            w = amask if edit_mask is None else amask * (edit_mask.float().cpu() * self.fg + (1 - edit_mask.float().cpu()) * self.bg)
            norm = 1.0 / (C * (float(sum(lt)) + 1e-12))
            return (x0, ctrl, pe, shapes, noise.to(dev, BF), sigma, w.to(dev).contiguous(), norm, (Lt, Lc, Ltot, txt_len))
        w, norm = self._dense_loss_weights(B, L, C, edit_mask)
        return (x0, ctrl, pe, shapes, noise.to(dev, BF), sigma, w, norm)

    # --------------------------------------------------------------------------------------------- public
    def compute_loss(self, embeddings: dict, noise=None, u=None) -> torch.Tensor:
        """Drop-in for `Trainer._compute_loss(embeddings)`: scalar loss whose `.backward()` fills the LoRA `.grad`s."""
        return self._autograd_loss(self._prepare(embeddings, noise, u))

    @torch.no_grad()
    def train_step(self, embeddings: dict, optimizer=None, noise=None, u=None):
        """Fast path (no autograd graph): fused fwd/loss/bwd -> NCCL mean all-reduce of the flat LoRA gradient ->
        clip -> bf16 grads -> optimizer.step().  Returns the (device) loss tensor; nothing here syncs with the host."""
        return self._fused_micro_step(self._prepare(embeddings, noise, u), optimizer)


class FluxKontextStep(_FusedStep):
    """Mirror of `FluxKontextLoraTrainer._compute_loss_shared_mode`
    (/root/reference/src/qflux/trainer/flux_kontext_trainer.py:494-577): t ~ U(0,1) in bf16 on the device, x_t = (1-t) x0 + t eps,
    ids = [target ids ; control ids], guidance = 1 when the model has guidance embeddings, target = eps - x0, MSE."""

    @staticmethod
    def latent_image_ids(h2, w2, device, first=0.0):
        """_prepare_latent_image_ids (flux_kontext_trainer.py:869-883): [h2*w2, 3] = (first, row, col)."""
        ids = torch.zeros(h2, w2, 3, device=device)
        ids[..., 0] = first
        ids[..., 1] = ids[..., 1] + torch.arange(h2, device=device)[:, None]
        ids[..., 2] = ids[..., 2] + torch.arange(w2, device=device)[None, :]
        return ids.reshape(h2 * w2, 3)

    def _prepare(self, embeddings, noise, t):
        m = self.dit
        dev = m.dev
        x0 = embeddings["image_latents"].to(dev, BF, non_blocking=True).contiguous()
        ctrl = embeddings["control_latents"].to(dev, BF, non_blocking=True).contiguous()
        pe = embeddings["prompt_embeds"].to(dev, BF, non_blocking=True).contiguous()
        pooled = embeddings["pooled_prompt_embeds"].to(dev, BF, non_blocking=True).contiguous()
        B, L, C = x0.shape
        if noise is None:
            noise = embeddings["noise"] if "noise" in embeddings else torch.randn(x0.shape, device=dev, dtype=BF)
        if t is None:
            t = embeddings["timestep"] if "timestep" in embeddings else torch.rand((B,), device=dev, dtype=BF)
        t = t.to(dev, BF)
        edit_mask = embeddings.get("edit_mask")
        shapes = embeddings.get("img_shapes")
        if shapes is not None and any(list(map(tuple, sh)) != list(map(tuple, shapes[0])) for sh in shapes):
            return self._prepare_multi(embeddings, x0, ctrl, pe, pooled, noise.to(dev, BF), t, edit_mask, shapes)
        ids = torch.cat([embeddings["image_ids"].to(dev), embeddings["control_ids"].to(dev)], dim=0)
        w, norm = self._dense_loss_weights(B, L, C, edit_mask)
        guidance = torch.ones(B, device=dev) if m.config.guidance_embeds else None
        return (x0, ctrl, pe, pooled, embeddings["text_ids"].to(dev), ids, noise.to(dev, BF), t, guidance, w, norm)

    def _prepare_multi(self, embeddings, x0, ctrl, pe, pooled, noise, t, edit_mask, shapes):
        """`_compute_loss_multi_resolution_mode` (flux_kontext_trainer.py:579-796): img_shapes is one list per sample of
        latent-patch shapes [(1, h, w) target, (1, h, w) control_1, ...] (the trainer converts pixel shapes with
        convert_img_shapes_to_latent first); image / control latents are zero-padded to the batch maximum.  Per-sample ids
        (control j carries j in the first column, :635-650), sequences [target | controls] padded to the longest sample, key mask,
        and a loss over the valid target tokens only.  All bookkeeping is host metadata: no device sync."""
        m, dev = self.dit, self.dit.dev
        B, L, C = x0.shape
        T = pe.shape[1]
        lt, lc, Ltot, Lt, Lc, amask = self._var_lengths(shapes, L)
        ids = torch.zeros(B, Ltot, 3)
        for b, sh in enumerate(shapes):
            parts = [self.latent_image_ids(sh[0][1], sh[0][2], "cpu", 0.0)]
            parts += [self.latent_image_ids(h, w_, "cpu", float(j + 1)) for j, (_, h, w_) in enumerate(sh[1:])]
            cat = torch.cat(parts, dim=0)
            ids[b, : cat.shape[0]] = cat
        kv_len = torch.tensor([T + a + b for a, b in zip(lt, lc)], dtype=torch.int32).to(dev, non_blocking=True)
        w = amask
        if edit_mask is not None and self.loss_kind != "mse":
            em = edit_mask.float().cpu()
            w = amask * (em * self.fg + (1 - em) * self.bg)
        # MseLoss ignores the mask: mean over all B*L*C elements, padded ones contribute 0 (prediction and target are both zero
        # there); AttentionMaskMseLoss divides by the valid-token count (attention_mask_loss.py:146-226)
        norm = 1.0 / (C * (float(sum(lt)) + 1e-12)) if self.loss_kind == "attention_mask" else 1.0 / (B * L * C)
        guidance = torch.ones(B, device=dev) if m.config.guidance_embeds else None
        return (x0, ctrl, pe, pooled, embeddings["text_ids"].to(dev), ids.to(dev, non_blocking=True), noise, t, guidance,
                w.to(dev).contiguous(), norm, (Lt, Lc, Ltot, kv_len, tuple(a + b for a, b in zip(lt, lc))))

    def _run(self, x0, ctrl, pe, pooled, text_ids, ids, noise, t, guidance, w, norm, var=None):
        m = self.dit
        B, L, C = x0.shape
        if var is None:
            packed = torch.empty(B, L + ctrl.shape[1], C, device=m.dev, dtype=BF)
            lib.flow_noisy_input(x0, noise, ctrl, t.float().contiguous(), packed)
            pred = m._forward_impl(packed, pe, pooled, t, ids, text_ids, guidance, train=True)
        else:
            Lt, Lc, Ltot, kv_len, valid_rows = var  # valid_rows: host copy of kv_len - T (plans the ragged GEMM row bands; part of the graph key)
            packed = torch.empty(B, Ltot, C, device=m.dev, dtype=BF)
            lib.flow_noisy_input_var(x0, noise, ctrl, t.float().contiguous(), Lt, Lc, packed)
            pred = m._forward_impl(packed, pe, pooled, t, ids, text_ids, guidance, kv_len, train=True, valid_rows=valid_rows)
        return self._loss_and_backward(pred, x0, noise, w, norm)

    def compute_loss(self, embeddings: dict, noise=None, t=None) -> torch.Tensor:
        return self._autograd_loss(self._prepare(embeddings, noise, t))

    @torch.no_grad()
    def train_step(self, embeddings: dict, optimizer=None, noise=None, t=None):
        return self._fused_micro_step(self._prepare(embeddings, noise, t), optimizer)
