"""Glue between the reference's trainer objects and the fused B200 path (SURVEY.md §7 step 2, §8b): nothing here computes.

    from qflux_b200 import patch_trainer
    trainer.load_model(); ...                     # the reference's own code, unchanged
    patch_trainer(trainer)                        # self.dit -> QwenImageB200 / FluxB200 (same weights), _compute_loss -> fused step

After the patch the reference's loop body runs as written (/root/reference/src/qflux/trainer/base_trainer.py:518-536):
`training_step -> _compute_loss` returns a scalar whose `.backward()` publishes the fused LoRA gradients into `param.grad`,
`accelerator.backward`, `clip_gradients`, `optimizer.step`, `lr_scheduler.step`, `zero_grad`, `save_lora` and
`get_lora_layers(self.dit)` all operate on ordinary `nn.Parameter`s with PEFT's names.
"""
from __future__ import annotations

import torch

_LOSS_KIND = {"MseLoss": "mse", "MaskEditLoss": "mask_edit", "AttentionMaskMseLoss": "attention_mask"}


def _cfg_get(cfg, k, default=None):
    try:
        return cfg[k]
    except (KeyError, TypeError, AttributeError):
        return getattr(cfg, k, default)


def from_reference(ref_model, device=None, _host_only: bool = False, frozen_weights=None):
    """Build the fused model for a loaded reference / diffusers transformer (`QwenImageTransformer2DModel` or
    `FluxTransformer2DModel`): same config, weights copied through the shared state-dict key names, and — when the module already
    carries a PEFT adapter (`peft_config`) — the same adapter with the same factors.  A 4-bit base model (bitsandbytes `Linear4bit`,
    NF4) gives a model whose block matrices stay NF4-resident (`frozen_weights`, picked per stacked kind from what the state dict holds).
    frozen_weights="fp8" keeps the block matrices of a float8-e4m3fn checkpoint FP8-resident; they may arrive as float8_e4m3fn or as
    the exact bf16 upcast that diffusers' `from_pretrained(torch_dtype=bfloat16)` holds (fp8.py).  Any other value is passed to the
    constructor as given."""
    from . import nf4
    from .flux_model import FluxB200, FluxB200Config
    from .qwen_model import QwenB200Config, QwenImageB200
    cfg = ref_model.config
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device()) if not _host_only else torch.device("cpu")
    is_flux = _cfg_get(cfg, "num_single_layers") is not None
    C, M = (FluxB200Config, FluxB200) if is_flux else (QwenB200Config, QwenImageB200)
    kw = {k: _cfg_get(cfg, k) for k in C.__dataclass_fields__ if _cfg_get(cfg, k) is not None}
    kw["axes_dims_rope"] = tuple(kw.get("axes_dims_rope", (16, 56, 56)))
    sd = ref_model.state_dict()
    plain, quant = nf4.split_state_dict(sd)
    nf4_kw = {}
    if quant:
        kinds, sizes = {}, set()
        for k, q in quant.items():
            kk = k.replace(".base_layer.", ".")
            kind = M._matrix_kind(kk[len("transformer."):] if kk.startswith("transformer.") else kk)
            if kind is not None:
                kinds[kind] = k
                sizes.add(q.blocksize)
        if len(sizes) > 1:
            raise nf4.QfxError(f"the NF4 block matrices use blocksizes {sorted(sizes)}; the fused layout takes one per model")
        if kinds:
            nf4_kw = dict(frozen_weights=tuple(kinds), nf4_blocksize=sizes.pop())
    if frozen_weights is not None:
        nf4_kw["frozen_weights"] = frozen_weights
    dit = M(C(**kw), device=device, _host_only=_host_only, **nf4_kw)
    peft_cfg = getattr(ref_model, "peft_config", None)
    if peft_cfg:
        (name, pc), = list(peft_cfg.items())
        dit.add_adapter(pc, adapter_name=name)
    if dit.frozen_weights == "fp8":
        dit.load_state_dict(sd, strict=True)
    elif quant or dit.frozen_weights != "bf16":
        dit._load_nf4(plain, quant, strict=True)
    else:
        dit.load_state_dict(sd, strict=True)
    return dit


def patch_trainer(trainer, use_fused_step: bool = True, _host_only: bool = False):
    """Swap the hot path of a constructed reference trainer (QwenImageEdit / QwenImageEditPlus / FluxKontext) in place.

    * `trainer.dit` becomes the fused model (weights and adapter taken over from the loaded reference module), with FP8-resident
      block weights when the trainer's config reports `quantization_type == "pretrain_fp8"` (the reference's marker of an FP8
      checkpoint, config.py `_compute_quantization_type`);
    * `trainer._compute_loss(embeddings)` becomes `QwenImageEditStep.compute_loss` / `FluxKontextStep.compute_loss` (same contract:
      scalar with autograd history to the LoRA parameters), with the loss kind read off `trainer.criterion`;
    * `trainer.b200_step` exposes the fused step for callers that want the no-autograd fast path (`train_step`).
    Returns the trainer."""
    from .flux_model import FluxB200
    from .mmdit_base import FusedMMDiTBase
    from .train_step import FluxKontextStep, QwenImageEditStep
    dit = trainer.dit
    if not isinstance(dit, FusedMMDiTBase):
        acc = getattr(trainer, "accelerator", None)
        fw = "fp8" if _cfg_get(getattr(trainer, "config", None), "quantization_type") == "pretrain_fp8" else None
        dit = from_reference(dit, getattr(acc, "device", None), _host_only, frozen_weights=fw)
        trainer.dit = dit
    crit = getattr(trainer, "criterion", None)
    kind = _LOSS_KIND.get(type(crit).__name__, "mse")
    fg = getattr(crit, "foreground_weight", getattr(crit, "forground_weight", 2.0))
    bg = getattr(crit, "background_weight", 1.0)
    tc = getattr(getattr(trainer, "config", None), "train", None)
    mgn = getattr(tc, "max_grad_norm", 1.0)
    gas = getattr(tc, "gradient_accumulation_steps", 1)
    if isinstance(dit, FluxB200):
        step = FluxKontextStep(dit, kind, fg=fg, bg=bg, max_grad_norm=mgn, gradient_accumulation_steps=gas)
        to_emb = _flux_embeddings(trainer)
    else:
        step = QwenImageEditStep(dit, kind, fg=fg, bg=bg, max_grad_norm=mgn, gradient_accumulation_steps=gas)
        to_emb = lambda e: e
    trainer.b200_step = step
    if use_fused_step:
        trainer._compute_loss = lambda embeddings, _s=step, _f=to_emb: _s.compute_loss(_f(embeddings))
    return trainer


def _flux_embeddings(trainer):
    """The FLUX trainer derives the target ids from the pixel image shape and passes pixel-space `img_shapes`
    (flux_kontext_trainer.py:494-577, 579-650); the fused step takes ids / latent-patch shapes."""
    from .train_step import FluxKontextStep
    vsf = getattr(trainer, "vae_scale_factor", 8)

    def conv(e):
        e = dict(e)
        if "image_ids" not in e and "image" in e:
            h, w = (int(s) // (vsf * 2) for s in e["image"].shape[2:])
            e["image_ids"] = FluxKontextStep.latent_image_ids(h, w, "cpu", 0.0)
        sh = e.get("img_shapes")
        if sh is not None and len(sh) and len(sh[0]) and sh[0][0][0] == 3:  # (C, H, W) pixels -> (1, H/16, W/16) latent patches
            e["img_shapes"] = [[(1, int(H) // (vsf * 2), int(W) // (vsf * 2)) for (_, H, W) in s] for s in sh]
        return e
    return conv
