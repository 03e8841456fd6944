"""ORACLE — test infrastructure only.  Block-streamed versions of `mmdit_oracle.QwenImageOracle` and `FluxOracle` for full-depth models.

A full-depth oracle in fp32 or fp64 does not fit an 80 GB device (the 60 Qwen-Image blocks alone are 82 GB in fp32), so this module
keeps only what is small resident and streams the blocks:

  * the top-level module IS the existing oracle class, built with its non-block parts (embedders, `txt_norm`, time / text embedding,
    `norm_out`, `proj_out`) and their LoRA adapters, loaded from the fused model's `state_dict()` in the oracle dtype;
  * every entry of `transformer_blocks` / `single_transformer_blocks` is a `StreamedBlock`.  It holds that block's LoRA factors as
    persistent leaves in the oracle dtype (so `.grad` accumulates on them across samples) and the fused model's views of the block's
    frozen weights.  Its forward runs `torch.utils.checkpoint` around `build()` + the block call: `build()` materialises an
    `mmdit_oracle.QwenBlock` / `FluxDoubleBlock` / `FluxSingleBlock` on the meta device, attaches empty PEFT adapters, and loads it
    strictly (`assign=True`) from the block's weights cast to the oracle dtype plus the persistent LoRA leaves.  The block is dropped
    after the call; the backward rebuilds it from the same weights.

No block math is restated here: the block classes, the top-level forwards and the loss recipes are those of mmdit_oracle.  The weights
are read when a block is built, so the oracle always sees the fused model's current frozen weights; the LoRA factors are copied once,
when the oracle is made.
"""
from __future__ import annotations

import functools

import torch
import torch.nn as nn
from torch.utils.checkpoint import checkpoint

from oracle import mmdit_oracle as mo

_BLOCK_LISTS = ("transformer_blocks", "single_transformer_blocks")


def _register(root: nn.Module, dotted: str, p: nn.Parameter):
    """Register `p` at the dotted path under `root`, creating empty modules on the way (names like `to_out.0` included)."""
    parts = dotted.split(".")
    mod = root
    for part in parts[:-1]:
        if part not in mod._modules:
            mod.add_module(part, nn.Module())
        mod = mod._modules[part]
    mod.register_parameter(parts[-1], p)


def _attach_adapter(mod: mo.LoraLinear, r: int, scaling: float, device="meta"):
    """A PEFT adapter with placeholder factors on a LoraLinear (the layout of `LoraLinear.add_adapter`; the factors are loaded next)."""
    mod.lora_A["default"] = nn.Linear(mod.in_features, r, bias=False, device=device)
    mod.lora_B["default"] = nn.Linear(r, mod.out_features, bias=False, device=device)
    mod.r, mod.scaling = r, scaling


def _lora_modules(keys) -> list[str]:
    return sorted({k.rsplit(".lora_A.", 1)[0] for k in keys if ".lora_A." in k})


class StreamedBlock(nn.Module):
    """One transformer block of a streamed oracle: LoRA leaves resident, frozen weights read from the fused model on every build."""

    def __init__(self, make, weights: dict, lora: dict, rank: int, scaling: float, dtype, device, prefix: str):
        """make: builds the oracle block class (called under the meta device); weights: block-relative key -> fused model tensor;
        lora: block-relative LoRA key -> tensor (copied into a persistent leaf)."""
        super().__init__()
        self._make, self._dtype, self._device = make, dtype, torch.device(device)
        self._weights = dict(weights)  # a plain dict: not parameters of this module, never moved or saved with it
        self._rank, self._scaling = rank, scaling
        self.prefix = prefix
        for k, v in lora.items():
            _register(self, k, nn.Parameter(v.detach().to(self._device, dtype).clone()))

    def source_keys(self) -> list[str]:
        """The fused model's state-dict keys this block is built from (frozen weights and LoRA factors)."""
        return [self.prefix + k for k in self._weights] + [self.prefix + n for n, _ in self.named_parameters()]

    def build(self) -> nn.Module:
        with torch.device("meta"):
            blk = self._make()
        blk.requires_grad_(False)
        lora = dict(self.named_parameters())
        for name in _lora_modules(lora):
            _attach_adapter(blk.get_submodule(name), self._rank, self._scaling)
        sd = {k: v.to(self._device, self._dtype) for k, v in self._weights.items()}
        sd.update(lora)
        blk.load_state_dict(sd, strict=True, assign=True)  # every weight of the block comes from the fused model, each key once
        return blk

    def _run(self, *args):
        return self.build()(*args)

    def forward(self, *args):
        return checkpoint(self._run, *args, use_reentrant=False)


def _split(sd: dict):
    """(top-level entries, {(list name, index): {block-relative key: tensor}}) of a fused state dict."""
    top, blocks = {}, {}
    for k, v in sd.items():
        head = k.split(".", 2)
        if head[0] in _BLOCK_LISTS:
            blocks.setdefault((head[0], int(head[1])), {})[head[2]] = v
        else:
            top[k] = v
    return top, blocks


def _streamed(orc_cls, cfg, fused, dtype, device, makers: dict):
    """Common part of `streamed_qwen` / `streamed_flux`: the oracle class with no blocks, its LoRA adapters and weights, then one
    StreamedBlock per fused block.  makers: list name -> (number of blocks, block constructor)."""
    device = torch.device(device)
    sd = fused.state_dict()
    top, blocks = _split(sd)
    r, scaling = fused.lora_rank, fused.lora_scaling
    o = orc_cls(cfg)  # on the host: its non-block parts are small, and it builds host-side tables (Qwen's RoPE) at construction
    o.requires_grad_(False)
    for name in _lora_modules(top):
        _attach_adapter(o.get_submodule(name), r, scaling, "cpu")
    o = o.to(device, dtype)
    o.load_state_dict({k: v.to(device, dtype) for k, v in top.items()}, strict=True)
    for n, p in o.named_parameters():
        p.requires_grad_("lora" in n)
    o.stream_top_keys = sorted(top)
    for lst, (n, make) in makers.items():
        mods = []
        for l in range(n):
            ent = blocks.pop((lst, l))
            lora = {k: v for k, v in ent.items() if ".lora_" in k}
            weights = {k: v for k, v in ent.items() if ".lora_" not in k}
            mods.append(StreamedBlock(make, weights, lora, r, scaling, dtype, device, f"{lst}.{l}."))
        setattr(o, lst, nn.ModuleList(mods))
    if blocks:
        raise KeyError(f"state-dict blocks the oracle has no place for: {sorted(blocks)[:4]}")
    return o


def streamed_qwen(fused, dtype=torch.float64, device=None) -> mo.QwenImageOracle:
    """`QwenImageOracle` of the fused Qwen-Image model `fused`, blocks streamed, in `dtype` on `device` (default: the model's)."""
    c = fused.config
    cfg = mo.QwenConfig(patch_size=c.patch_size, in_channels=c.in_channels, out_channels=c.out_channels, num_layers=0,
                        attention_head_dim=c.attention_head_dim, num_attention_heads=c.num_attention_heads,
                        joint_attention_dim=c.joint_attention_dim, guidance_embeds=c.guidance_embeds, axes_dims_rope=tuple(c.axes_dims_rope))
    D, H = fused.D, fused.H
    o = _streamed(mo.QwenImageOracle, cfg, fused, dtype, device or fused.dev,
                  {"transformer_blocks": (fused.L, functools.partial(mo.QwenBlock, D, H, c.attention_head_dim))})
    o.config.num_layers = fused.L
    return o


def streamed_flux(fused, dtype=torch.float64, device=None) -> mo.FluxOracle:
    """`FluxOracle` of the fused FLUX model `fused`, double and single blocks streamed, in `dtype` on `device`."""
    c = fused.config
    cfg = mo.FluxConfig(patch_size=c.patch_size, in_channels=c.in_channels, out_channels=c.out_channels, num_layers=0,
                        num_single_layers=0, attention_head_dim=c.attention_head_dim, num_attention_heads=c.num_attention_heads,
                        joint_attention_dim=c.joint_attention_dim, pooled_projection_dim=c.pooled_projection_dim,
                        guidance_embeds=c.guidance_embeds, axes_dims_rope=tuple(c.axes_dims_rope))
    D, H, hd = fused.D, fused.H, c.attention_head_dim
    o = _streamed(mo.FluxOracle, cfg, fused, dtype, device or fused.dev,
                  {"transformer_blocks": (fused.L, functools.partial(mo.FluxDoubleBlock, D, H, hd)),
                   "single_transformer_blocks": (fused.Ls, functools.partial(mo.FluxSingleBlock, D, H, hd))})
    o.config.num_layers, o.config.num_single_layers = fused.L, fused.Ls
    return o


def streamed_oracle(fused, dtype=torch.float64, device=None):
    """The streamed oracle of either model family."""
    return (streamed_flux if hasattr(fused.config, "pooled_projection_dim") else streamed_qwen)(fused, dtype, device)


def source_keys(o) -> list[str]:
    """Every fused state-dict key the streamed oracle `o` is built from, once per use (top level, then each block)."""
    keys = list(o.stream_top_keys)
    for lst in _BLOCK_LISTS:
        for blk in getattr(o, lst, ()):
            keys += blk.source_keys()
    return keys
