"""Shared host-side machinery of the fused B200 MMDiT models (Qwen-Image, FLUX): HBM layout, LoRA registry, sharded frozen
weights, the double-stream block forward/backward launch sequences, the block stack with its output head, the CUDA-graph cache
and the autograd bridge.  All arithmetic is in libqfx_b200.so.

Layout conventions (DESIGN.md §3):
  * tokens are stream-major: rows [0, B*T) text (stream index 1), rows [B*T, B*T + B*L) image (stream index 0);
  * frozen weights are plain device tensors in `self.w`, layer-stacked and fused (q|k|v concatenated per stream);
  * a "site" is one (block, weight group, stream) that may carry LoRA factors, zero-padded to Rp = 64 * ceil(r / 64) (`A_pad [Rp*n, in]`,
    `B_pad [n*out, Rp]`, n = 3 for a fused q|k|v site); the trainable nn.Parameters are views into those buffers;
  * LoRA gradients accumulate in one flat fp32 buffer `G32` (the all-reduce payload); `G16` holds the bf16 grads.
"""
from __future__ import annotations

import math
import numbers
import os
import re
import warnings
from typing import NamedTuple

import torch
import torch.distributed as dist
import torch.nn as nn

from . import lib

BF = torch.bfloat16
PAD = 64  # width of one k-block of the fused GEMM; the LoRA rank is padded to Rp = PAD * ceil(r / PAD) (one or two k-blocks)
MAX_RANK = 128
NARROW_RANKS = (64, 32, 16, 8, 4)  # the ranks qfx_lora_wgrad takes (the 64-channel embedder's dA runs in chunks of these widths)
DEFAULT_TARGETS = ("to_q", "to_k", "to_v", "to_out.0")  # /root/reference/src/qflux/data/config.py:315
# Device memory left free when the training workspace is planned (the default activation limit is the free device memory minus this):
# what a step allocates after its workspace.  Measured with tools/recompute_bench.py on an H100 80GB HBM3 (400 W), every Qwen-Image-Edit,
# Edit-Plus and FLUX-Kontext point: the step's peak exceeded "allocated when planned + workspace" by at most 0.36 GiB (the captured
# step graph's pool, step temporaries) and the allocator's reserved memory by at most 0.93 GiB.  The rest of the 4 GiB is left for
# what that run did not allocate after its workspace: fused-AdamW moments of an optimizer built after the first step and the no-grad
# workspaces of a validation pass (a few hundred MB each, up to three).
ACTIVATION_HEADROOM = 4 << 30


def padded_rank(r: int) -> int:
    """Rp: the rank's columns in the padded factor buffers and the T / U workspaces."""
    return PAD * -(-r // PAD)


def check_rank(r) -> None:
    """The fused path's rank rule: one rank for every adapted module, a multiple of 4 from 4 to MAX_RANK."""
    if isinstance(r, bool) or not isinstance(r, numbers.Integral) or not (4 <= r <= MAX_RANK and r % 4 == 0):
        raise NotImplementedError(f"LoRA rank {r!r}: the fused path takes one rank for every adapted module, a multiple of 4 from 4 "
                                  f"to {MAX_RANK}")


def rank_chunks(r: int):
    """(first rank, width) pieces of [0, r), widths from NARROW_RANKS, largest first: every first rank is a multiple of 8 unless r < 8."""
    out, c0 = [], 0
    while c0 < r:
        w = next(w for w in NARROW_RANKS if w <= r - c0)
        out.append((c0, w))
        c0 += w
    return out


class ActivationPlan(NamedTuple):
    """Which blocks of the training workspace keep their saved tensors (DESIGN.md §3).
    recompute: global block indices (double blocks first, then single blocks) that keep only their input X[blk] — the backward
    re-runs their forward into a scratch dict right before their backward; bytes: planned workspace bytes; saved_bytes: how many
    fewer bytes than keep-all; min_bytes: the bytes with every block recomputed; limit: the bytes the workspace was allowed
    (None: unlimited)."""
    recompute: tuple
    bytes: int
    saved_bytes: int
    min_bytes: int
    limit: int | None


def plan_activation_memory(blocks, fixed: int, limit: int | None) -> ActivationPlan:
    """blocks: one (kind, {saved entry: bytes}) per block in execution order; fixed: the workspace bytes every plan allocates.
    Keep-all when it fits `limit`, else recompute the fewest blocks, taken from the end of the stack.  The recomputed blocks of a
    kind share one scratch dict holding every entry any of them needs.  Raises QfxError when not even recomputing every block fits."""
    n = len(blocks)

    def total(k):
        scratch = {}
        for kind, ent in blocks[n - k:]:
            s = scratch.setdefault(kind, {})
            for name, b in ent.items():
                s[name] = max(s.get(name, 0), b)
        return fixed + sum(sum(e.values()) for _, e in blocks[:n - k]) + sum(sum(s.values()) for s in scratch.values())

    keep_all, least = total(0), total(n)
    for k in range(n + 1):
        t = total(k)
        if limit is None or t <= limit:
            return ActivationPlan(tuple(range(n - k, n)), t, keep_all - t, least, limit)
    raise lib.QfxError(f"the training workspace needs {least} bytes with the activations of every block recomputed, but only {limit} "
                       f"bytes are available for it (keeping every block would take {keep_all}): use a smaller batch or free device memory")


class LoraSite:
    """LoRA factors of one (block, group): padded buffers shared by its 1 or 3 member modules (and, for FLUX single
    blocks, by both streams)."""

    def __init__(self, n_slots, d_in, d_out_each, rp, device):
        self.n, self.rp = n_slots, rp
        self.A_pad = torch.zeros(n_slots * rp, d_in, device=device, dtype=BF)        # rows g*Rp.. = A of slot g
        self.B_pad = torch.zeros(n_slots * d_out_each, rp, device=device, dtype=BF)  # rows g*out.. = B of slot g
        self.members = {}  # slot -> (name, A_param, B_param, gA_off, gB_off, d_in, d_out)
        self.r = 0


class _LoraConfigLike:
    """The attributes of `peft.LoraConfig` this path reads and `get_peft_model_state_dict` inspects (used when peft is not installed
    or the short `add_adapter(r, alpha)` form is used)."""
    peft_type = "LORA"
    bias = "none"
    use_dora = False
    lora_dropout = 0.0
    layer_replication = None
    rank_pattern: dict = {}
    alpha_pattern: dict = {}
    is_prompt_learning = False

    def __init__(self, r, lora_alpha, target_modules, init_lora_weights="gaussian"):
        self.r, self.lora_alpha, self.target_modules, self.init_lora_weights = r, lora_alpha, target_modules, init_lora_weights

    def to_dict(self):
        return dict(r=self.r, lora_alpha=self.lora_alpha, target_modules=self.target_modules, init_lora_weights=self.init_lora_weights,
                    peft_type=self.peft_type, bias=self.bias)


class FusedMMDiTBase(nn.Module):
    # subclasses fill these -------------------------------------------------------------------------------------------
    round_mid = True  # diffusers RMSNorm (Qwen) rounds before the weight multiply; torch.nn.RMSNorm (FLUX) does not
    keep_qkv = True   # keep normalised/rotated Q,K,V and the LN1 output of double blocks for the backward (HBM for time)
    Ls = 0            # single-stream blocks (FLUX), run after the L double-stream blocks
    _DOUBLE_LINEARS: dict = {}  # diffusers sub-module name of a double-block Linear -> (group, stream, slot); stream 0 = image, 1 = text
    _ADALN = ("", "")           # sub-module names of a double block's (image, text) AdaLN modulation Linears
    _PER_LAYER = ("mod_w", "mod_b", "qkv_w", "qkv_b", "out_w", "out_b", "up_w", "up_b", "down_w", "down_b", "qknorm_w")
    _PER_SINGLE = ()
    _NF4_KINDS = ("mod_w", "qkv_w", "out_w", "up_w", "down_w")  # the stacked matrices a 4-bit base checkpoint keeps NF4-resident
    _SINGLE_MATS: dict = {}     # sub-module name of a single-block Linear -> its stacked kind (FLUX)
    _sharded_s = None           # the single blocks' sharded ring once shard_frozen_weights() has run

    def _weight_views(self) -> dict:
        raise NotImplementedError

    def _double_weight_views(self, out: dict, w: dict, blocks: bool) -> dict:
        """Adds the state-dict entries of every double block of `w` to `out` when `blocks` (block weights that come through a ring
        are not addressable as full tensors)."""
        D = self.D
        for l in range(self.L if blocks else 0):
            b = f"transformer_blocks.{l}."
            for s, nm in enumerate(self._ADALN):
                out[b + nm + ".weight"], out[b + nm + ".bias"] = w["mod_w"][l, s], w["mod_b"][l, s]
            for i, nm in enumerate(("attn.norm_q", "attn.norm_k", "attn.norm_added_q", "attn.norm_added_k")):
                out[b + nm + ".weight"] = w["qknorm_w"][l, i]
            for nm, (grp, s, slot) in self._DOUBLE_LINEARS.items():
                W, Bv = w[grp + "_w"][l, s], w[grp + "_b"][l, s]
                if grp == "qkv":
                    W, Bv = W[slot * D:(slot + 1) * D], Bv[slot * D:(slot + 1) * D]
                out[b + nm + ".weight"], out[b + nm + ".bias"] = W, Bv
        return out

    def _linear_table(self) -> dict:
        """full module name -> (site_key=(l, grp), streams tuple, slot, d_in, d_out, n_slots)"""
        D = self.D
        dims = {"qkv": (D, D, 3), "out": (D, D, 1), "up": (D, 4 * D, 1), "down": (4 * D, D, 1)}
        t = {}
        for l in range(self.L):
            for nm, (grp, s, slot) in self._DOUBLE_LINEARS.items():
                d_in, d_out, n = dims[grp]
                t[f"transformer_blocks.{l}.{nm}"] = ((l, grp), (s,), slot, d_in, d_out, n)
        return t

    def _mod_table(self) -> dict:
        """full name of an AdaLN modulation Linear -> (kind, index, n_chunks): kind "dbl" indexes rows of ws["mods"] viewed
        [B, L*2, 6D] (index = 2*l + stream), kind "sgl" rows of ws["smods"] viewed [B, Ls, 3D]."""
        t = {}
        for l in range(self.L):
            for s, nm in enumerate(self._ADALN):
                t[f"transformer_blocks.{l}.{nm}"] = ("dbl", 2 * l + s, 6)
        return t

    def _embed_table(self) -> dict:
        """full name of an input embedder Linear -> (weight key prefix in self.w, stream, d_in), image embedder first."""
        return {}

    def _wb(self, l, grp, s):
        if l < 0:  # input embedders: one weight, no block index
            return self.w[grp + "_w"], self.w[grp + "_b"]
        return self.w[grp + "_w"][l, s], self.w[grp + "_b"][l, s]

    def _view_source(self, store: bool):
        """(weights dict, whether block entries are included) for `_weight_views`.  store=True: every block, with the NF4- or
        FP8-resident kinds as meta tensors of their bf16 shape — their views' storage offsets address the resident storage
        (load_state_dict).  Sharded weights have no addressable blocks either way."""
        if not store or self._sharded is not None:
            return self.w, self._blk_rings is None
        w = dict(self.w)
        for k, (codes, _) in self._nf4_store.items():
            w[k] = torch.empty(*codes.shape[:-1], codes.shape[-1] * 2, device="meta", dtype=BF)
        for k, codes in self._fp8_store.items():
            w[k] = torch.empty(*codes.shape, device="meta", dtype=BF)
        return w, True

    @classmethod
    def _matrix_kind(cls, key: str):
        """Stacked kind ("qkv_w", "s_mod_w", ...) of the block Linear whose weight is `key` (None: not a block matrix)."""
        m = re.fullmatch(r"(single_)?transformer_blocks\.\d+\.(.+)\.weight", key)
        if m is None:
            return None
        if m.group(1):
            return cls._SINGLE_MATS.get(m.group(2))
        if m.group(2) in cls._ADALN:
            return "mod_w"
        grp = cls._DOUBLE_LINEARS.get(m.group(2))
        return None if grp is None else grp[0] + "_w"

    # -----------------------------------------------------------------------------------------------------------------
    def _init_common(self, device, host_only, frozen_weights="bf16", nf4_blocksize=64):
        """frozen_weights: "bf16" (block weights resident in bf16), "nf4" (every stacked block matrix NF4-resident: a 4-bit base
        checkpoint) or the set of stacked kinds that are (`from_reference` picks what the checkpoint holds), or "fp8" (every stacked
        block matrix held as float8-e4m3fn bytes: an FP8 base checkpoint without scales)."""
        if not host_only and not torch.cuda.is_available():
            raise lib.QfxError(f"{type(self).__name__} needs a CUDA device (sm_90a); there is no CPU fallback")
        kinds = () if frozen_weights in ("bf16", "fp8") else self._NF4_KINDS if frozen_weights == "nf4" else tuple(frozen_weights)
        if isinstance(frozen_weights, str) and frozen_weights not in ("bf16", "nf4", "fp8") or not set(kinds) <= set(self._NF4_KINDS):
            raise lib.QfxError(f"frozen_weights={frozen_weights!r}: 'bf16', 'nf4', 'fp8' or a subset of {self._NF4_KINDS}")
        self._nf4_kinds, self.nf4_blocksize = tuple(k for k in self._NF4_KINDS if k in kinds), int(nf4_blocksize)
        self._nf4_store = {}     # NF4-resident kind -> (codes uint8 [L, ..., in/2], absmax fp32 [L, n/blocksize])
        self._nf4_rings = None   # sharding.Nf4Blocks of (double, single) blocks
        self._fp8_kinds = self._NF4_KINDS if frozen_weights == "fp8" else ()
        self._fp8_store = {}     # FP8-resident kind -> codes float8_e4m3fn [L, ..., out, in]
        self._expand_rings = None  # (double, single) rings that expand codes (Nf4Blocks / Fp8Blocks, or their sharded forms)
        self._blk_rings = None   # (double, single) rings the block weights come through: NF4 / FP8 expansion or sharding
        self.dev = torch.device(device)
        self.sites = {}          # (l, grp, s) -> LoraSite   (l = -1: input embedders)
        self.mod_sites = {}      # kind -> dict(idx=[row indices], names=[...], A=[n, r, D], B=[n, C, r], ga, gb)  (AdaLN linears)
        self._lora_params = {}   # PEFT name -> nn.Parameter
        self.lora_scaling, self.lora_rank, self.lora_rp = 0.0, 0, PAD
        self.adapter_name, self.peft_config = "default", {}
        self.G32 = self.G16 = None
        self._ws = self._ws_key = None
        self._train_ws, self._infer_ws = None, {}   # cached workspaces (see _get_workspace)
        self._rope_cache = {}
        self.gradient_checkpointing = False  # accepted for interface compatibility (see enable_gradient_checkpointing)
        self._activation_limit = None  # bytes the training workspace may take; None: free device memory - ACTIVATION_HEADROOM
        self._sharded = None     # the double blocks' sharded ring once shard_frozen_weights() has run (weights sharded across ranks):
                                 # sharding.ShardedBlocks, or ShardedNf4Blocks / ShardedFp8Blocks for NF4 / FP8 codes
        self._grad_exchange = None  # sharding.GradExchange of deterministic data-parallel steps (False: ranks not on one host)
        self._bands_cache = {}   # (valid image rows per sample, Limg) -> lib.RowBands (ragged GEMM row bands)
        self._infer_graphs, self.use_cuda_graph_inference = GraphCache(8, "the inference forward"), True  # see _infer
        self._fwd_gen = 0        # bumped by every forward: autograd nodes of an older forward refuse to run (their activations are gone)

    def _frozen(self, kind, *shape):
        """A stacked block matrix [L, ..., out, in]: bf16 zeros, or — NF4-resident — its codes and absmax (in `self._nf4_store`), or
        — FP8-resident — its e4m3fn codes (in `self._fp8_store`).  A resident kind's bf16 stack is never allocated and `self.w[kind]`
        becomes a ring view in `_finish_frozen`."""
        if kind in self._fp8_kinds:
            self._fp8_store[kind] = torch.zeros(*shape, device=self.dev, dtype=torch.uint8).view(torch.float8_e4m3fn)
            return None
        if kind not in self._nf4_kinds:
            return torch.zeros(*shape, device=self.dev, dtype=BF)
        if shape[-1] % self.nf4_blocksize:
            raise lib.QfxError(f"{kind}: NF4 blocksize {self.nf4_blocksize} does not divide in_features {shape[-1]}")
        n = math.prod(shape[1:])
        self._nf4_store[kind] = (torch.zeros(*shape[:-1], shape[-1] // 2, device=self.dev, dtype=torch.uint8),
                                 torch.zeros(shape[0], n // self.nf4_blocksize, device=self.dev, dtype=torch.float32))
        return None

    def _finish_frozen(self):
        """NF4- or FP8-resident kinds: one two-slot ring per block kind, filled by dequantizing (NF4) or expanding (FP8) a block
        right before it runs."""
        if not (self._nf4_kinds or self._fp8_kinds):
            return
        from .sharding import Fp8Blocks, Nf4Blocks
        rings = []
        for per, n in ((self._PER_LAYER, self.L), (self._PER_SINGLE, self.Ls)):
            if self._fp8_kinds:
                st = {k: self._fp8_store[k] for k in per if k in self._fp8_store}
                rings.append(Fp8Blocks(st, n) if st else None)
            else:
                st = {k: (*self._nf4_store[k], tuple(self._nf4_store[k][0].shape[1:-1]) + (self._nf4_store[k][0].shape[-1] * 2,))
                      for k in per if k in self._nf4_store}
                rings.append(Nf4Blocks(st, n, self.nf4_blocksize) if st else None)
            for k in st:
                self.w[k] = rings[-1].rings[k]
        self._expand_rings = self._blk_rings = tuple(rings)
        if self._nf4_kinds:
            self._nf4_rings = self._expand_rings

    @property
    def frozen_weights(self) -> str:
        """How the frozen block weights are stored: "bf16", "nf4" (NF4-resident, dequantized block by block) or "fp8"
        (float8-e4m3fn-resident, expanded block by block)."""
        return "fp8" if self._fp8_kinds else "nf4" if self._nf4_kinds else "bf16"

    @property
    def device(self):
        return self.dev

    @property
    def dtype(self):
        return BF

    def shard_frozen_weights(self, group=None, gather="auto"):
        """BASELINE config 4 (the reference's FSDP branch, base_trainer.py:333-382): keep 1/world of every double and every single
        block's frozen weights on this rank; a block's full weights are assembled in one of two ring buffers right before it runs —
        by copy-engine pulls from the peers' shards on one node, by an NCCL all-gather otherwise (sharding.py; one two-slot ring
        per block kind).  Call after the weights are loaded (collective).  LoRA factors, embedders and the output head stay
        replicated; `state_dict()` then only carries the replicated tensors and the LoRA parameters.

        An NF4- or FP8-resident model (frozen_weights="nf4" / "fp8") shards its codes instead, at world >= 2: each rank keeps 1/world
        of every block's packed code bytes, and a block is filled by gathering them into a staging slot and expanding them there
        (sharding.ShardedCodes); biases and norm weights stay replicated bf16.  With the peer gather its steps and inference
        forwards are still CUDA-graph replayed."""
        from .sharding import ShardedBlocks
        if self._sharded is not None:
            return self
        if self._nf4_kinds or self._fp8_kinds:
            return self._shard_code_rings(group, gather)
        self._sharded = ShardedBlocks({k: self.w[k] for k in self._PER_LAYER}, self.L, group, gather=gather)
        for k in self._PER_LAYER:
            self.w[k] = self._sharded.rings[k]
        if self.Ls:
            self._sharded_s = ShardedBlocks({k: self.w[k] for k in self._PER_SINGLE}, self.Ls, group, gather=gather)
            for k in self._PER_SINGLE:
                self.w[k] = self._sharded_s.rings[k]
        self._blk_rings = (self._sharded, self._sharded_s)
        if torch.cuda.is_available():
            torch.cuda.empty_cache()
        return self

    def _shard_code_rings(self, group, gather):
        """shard_frozen_weights of an NF4- or FP8-resident model: the expansion rings become sharded code rings (one per block kind),
        and the full code stacks are freed."""
        from .sharding import ShardedFp8Blocks, ShardedNf4Blocks
        fmt = "FP8" if self._fp8_kinds else "NF4"
        world = dist.get_world_size(group) if dist.is_initialized() else 1
        if world < 2:
            raise lib.QfxError(f"shard_frozen_weights: the frozen weights are {fmt}-resident (frozen_weights='{fmt.lower()}') and "
                               f"there is one rank: sharded {fmt} needs world >= 2 (one rank already holds the one copy of the codes)")
        if self._nf4_kinds and set(self._nf4_kinds) != set(self._NF4_KINDS):
            raise lib.QfxError(f"shard_frozen_weights: only the stacked kinds {self._nf4_kinds} are NF4-resident (the others bf16); "
                               f"sharded NF4 needs every stacked block matrix NF4-resident (frozen_weights='nf4')")
        src = [None if r is None else (r.codes, {k: v.shape for k, v in r.rings.items()}) for r in self._expand_rings]
        for r in filter(None, self._expand_rings):  # a ring and its views refer to each other: drop its buffers without waiting for gc
            r.codes = r.gbuf = None
        self._expand_rings = self._blk_rings = self._nf4_rings = None  # the old slots go back to the allocator before the new ones
        for _, shapes in filter(None, src):
            for k in shapes:
                self.w[k] = None
        rings = []
        for ent, n in zip(src, (self.L, self.Ls)):
            if ent is None:
                rings.append(None)
                continue
            codes, shapes = ent
            if self._fp8_kinds:
                ring = ShardedFp8Blocks({k: c for k, (c,) in codes.items()}, n, group, gather=gather)
            else:
                ring = ShardedNf4Blocks({k: (c, a, shapes[k]) for k, (c, a) in codes.items()}, n, self.nf4_blocksize, group,
                                        gather=gather)
            for k in shapes:
                self.w[k] = ring.rings[k]
            rings.append(ring)
        self._expand_rings = self._blk_rings = tuple(rings)
        if self._nf4_kinds:
            self._nf4_rings = self._expand_rings
        self._sharded, self._sharded_s = rings
        self._nf4_store, self._fp8_store = {}, {}
        if torch.cuda.is_available():
            torch.cuda.empty_cache()
        return self

    def _ring(self, blk):
        """(ring or None, local index) of global block `blk` (double blocks first, then single blocks)."""
        return (self._blk_rings[0], blk) if blk < self.L else (self._blk_rings[1], blk - self.L)

    def _acquire(self, blk, nxt):
        """Ringed weights: make block `blk` resident and start filling block `nxt` (if there is one)."""
        ring, l = self._ring(blk)
        if ring is not None:
            ring.acquire(l)
        if 0 <= nxt < self.L + self.Ls:
            r2, l2 = self._ring(nxt)
            if r2 is not None:
                r2.prefetch(l2)

    def _release(self, blk):
        ring, l = self._ring(blk)
        if ring is not None:
            ring.release(l)

    def _join_expand_rings(self):
        for ring in self._expand_rings or ():
            if ring is not None:
                ring.join()

    def _block_mods(self, ws, blk):
        """Ringed weights: the base modulation vectors of block `blk` (plus their LoRA), from its now resident weights."""
        D, w = self.D, self.w
        if blk < self.L:
            lib.gemv_act(ws["temb"], w["mod_w"][blk].view(2 * 6 * D, D), w["mod_b"][blk].view(-1),
                         ws["mods"][:, blk * 12 * D:(blk + 1) * 12 * D], act=1)
            self._mod_lora_fwd(ws, ws["temb"], ("dbl", (2 * blk, 2 * blk + 1)))
        else:
            l = blk - self.L
            lib.gemv_act(ws["temb"], w["s_mod_w"][l], w["s_mod_b"][l], ws["smods"][:, l * 3 * D:(l + 1) * 3 * D], act=1)
            self._mod_lora_fwd(ws, ws["temb"], ("sgl", (l,)))

    def enable_gradient_checkpointing(self, *args, **kwargs):
        """Accepted for the reference trainer's `gradient_checkpointing: True`.  It selects nothing: the training workspace always
        recomputes the activations of exactly those blocks whose saved tensors do not fit the device (`activation_plan`)."""
        self.gradient_checkpointing = True

    def set_activation_memory_limit(self, nbytes: int | None):
        """Bytes the training workspace may take (None: the free device memory when it is built, minus ACTIVATION_HEADROOM).
        Drops the cached training workspace; the next training step plans and allocates it again under the new limit."""
        self._activation_limit = None if nbytes is None else int(nbytes)
        if self._train_ws is not None and self._ws is self._train_ws[1]:
            self._ws = self._ws_key = None
        self._train_ws = None

    @property
    def activation_plan(self) -> ActivationPlan | None:
        """The plan of the current training workspace (None before the first training step)."""
        return None if self._train_ws is None else self._train_ws[1]["plan"]

    def _apply(self, fn, recurse=True):
        """`dit.to(accelerator.device)` / `.cuda()` / `.bfloat16()` (base_trainer.py:388, qwen_image_edit_trainer.py:300-330) are accepted
        when they are no-ops; the HBM layout (fused, layer-stacked weights; LoRA parameters that are views into padded buffers) cannot be
        moved or re-typed tensor by tensor, so anything else fails loudly instead of silently detaching the views."""
        probe = torch.empty(0, device=self.dev, dtype=BF)
        moved = fn(probe)
        if moved.device != probe.device or (moved.dtype != BF and moved.is_floating_point()):
            raise lib.QfxError(f"{type(self).__name__} lives on {self.dev} in bf16; construct it on the target device instead of "
                               f"moving it (requested {moved.device}, {moved.dtype})")
        return self

    def zero_grad(self, set_to_none: bool = True):
        if self.G32 is not None:
            self.G32.zero_()
        for p in self.parameters():
            p.grad = None

    # ------------------------------------------------------------------------------------------------ state dict
    def state_dict(self, *args, **kwargs):
        """diffusers / PEFT key names; LoRA'd modules expose `base_layer.*` and `lora_{A,B}.default.weight`."""
        lora_mods = {n.rsplit(".lora_", 1)[0] for n in self._lora_params}
        sd = {}
        for k, v in self._weight_views().items():
            mod, leaf = k.rsplit(".", 1)
            sd[(mod + ".base_layer." + leaf) if mod in lora_mods else k] = v
        for k, p in self._lora_params.items():
            # lora_B parameters are strided views into the padded factor buffer: hand out compact copies (safetensors refuses
            # non-contiguous tensors, torch.save would serialise the whole padded storage)
            sd[k] = p.detach().contiguous().clone()
        return sd

    @torch.no_grad()
    def load_state_dict(self, sd, strict=True, assign=False):
        """bf16 checkpoints, and 4-bit NF4 base checkpoints (bitsandbytes `Linear4bit` entries, nf4.py): NF4 block matrices go to the
        NF4-resident storage of a model constructed with frozen_weights='nf4' (`from_reference` does), NF4 tensors outside the blocks
        are dequantized to bf16 here.  Into a model constructed with frozen_weights='fp8': block matrices as float8_e4m3fn or as their
        exact bf16 upcast (fp8.py).  A float8 tensor anywhere else, or into a bf16 model, is upcast to bf16."""
        from . import nf4
        plain, quant = nf4.split_state_dict(sd)
        if self._fp8_kinds:
            return self._load_fp8(plain, quant, strict)
        if quant or self._nf4_kinds:
            return self._load_nf4(plain, quant, strict)
        views = self._weight_views()
        unexpected, seen = [], set()
        for k, v in sd.items():
            kk = k.replace(".base_layer.", ".")
            lk = self._canonical_lora_key(k)
            if kk in views:
                views[kk].copy_(v.to(self.dev, BF))
                seen.add(kk)
            elif lk in self._lora_params:
                self._lora_params[lk].copy_(v.to(self.dev, BF))
                seen.add(lk)
            else:
                unexpected.append(k)
        missing = [k for k in list(views) + list(self._lora_params) if k not in seen]
        if strict and (unexpected or [m for m in missing if "lora" not in m]):
            raise KeyError(f"load_state_dict: missing {missing[:5]}..., unexpected {unexpected[:5]}...")
        return missing, unexpected

    def _load_nf4(self, plain, quant, strict):
        """load_state_dict of a checkpoint with NF4 entries or into an NF4-resident model: every block entry is addressable here
        (meta views stand for the NF4 kinds; a view's storage offset locates its rows in the codes / absmax stacks)."""
        from . import nf4
        views = self._weight_views(store=True)
        unexpected, seen = [], set()

        def canon(k):
            k = k.replace(".base_layer.", ".")
            return k[len("transformer."):] if k.startswith("transformer.") and k[len("transformer."):] in views else k

        for k, v in plain.items():
            kk, lk = canon(k), self._canonical_lora_key(k)
            if kk in views:
                if views[kk].is_meta:
                    raise lib.QfxError(f"`{kk}` arrives in bf16, but {self._matrix_kind(kk)} is NF4-resident in this model "
                                       f"(frozen_weights={self._nf4_kinds!r}): the layers of a stacked kind must arrive in one format; "
                                       f"construct with frozen_weights='bf16' for a bf16 checkpoint")
                views[kk].copy_(v.to(self.dev, BF))
                seen.add(kk)
            elif lk in self._lora_params:
                self._lora_params[lk].copy_(v.to(self.dev, BF))
                seen.add(lk)
            else:
                unexpected.append(k)
        for k, q in quant.items():
            kk = canon(k)
            if kk not in views:
                unexpected.append(k)
                continue
            t = views[kk]
            if tuple(t.shape) != q.shape:
                raise lib.QfxError(f"`{kk}`: NF4 shape {q.shape}, the model expects {tuple(t.shape)}")
            if not t.is_meta:
                if self._matrix_kind(kk) is not None:
                    raise lib.QfxError(f"`{kk}` is NF4 but this model keeps {self._matrix_kind(kk)} in bf16 (frozen_weights="
                                       f"{'bf16' if not self._nf4_kinds else self._nf4_kinds!r}): construct it with frozen_weights='nf4' "
                                       f"(from_reference does) for a 4-bit base checkpoint")
                t.copy_(nf4.dequantize(q).to(self.dev))  # outside the blocks: bf16 in the existing layout
            else:
                if q.blocksize != self.nf4_blocksize:
                    raise lib.QfxError(f"`{kk}`: NF4 blocksize {q.blocksize}, the model was constructed with nf4_blocksize="
                                       f"{self.nf4_blocksize}")
                codes, absmax = self._nf4_store[self._matrix_kind(kk)]
                o, n = t.storage_offset(), t.numel()
                codes.view(-1)[o // 2:(o + n) // 2].copy_(q.codes.to(self.dev))
                absmax.view(-1)[o // q.blocksize:(o + n) // q.blocksize].copy_(q.absmax.to(self.dev))
            seen.add(kk)
        missing = [k for k in list(views) + list(self._lora_params) if k not in seen]
        if strict and (unexpected or [m for m in missing if "lora" not in m]):
            raise KeyError(f"load_state_dict: missing {missing[:5]}..., unexpected {unexpected[:5]}...")
        return missing, unexpected

    def _load_fp8(self, plain, quant, strict):
        """load_state_dict into an FP8-resident model: a block matrix goes to the e4m3fn stack of its kind (a meta view's storage
        offset locates its elements), after fp8.as_e4m3 has checked it; every other entry loads as into a bf16 model."""
        from . import fp8
        if quant:
            raise lib.QfxError(f"`{next(iter(quant))}` is a bitsandbytes NF4 weight, but this model keeps its block matrices FP8-resident "
                               f"(frozen_weights='fp8'): construct it with frozen_weights='nf4' (from_reference does) for a 4-bit base "
                               f"checkpoint")
        views = self._weight_views(store=True)
        unexpected, seen, form = [], set(), {}

        def canon(k):
            k = k.replace(".base_layer.", ".")
            return k[len("transformer."):] if k.startswith("transformer.") and k[len("transformer."):] in views else k

        for k, v in plain.items():
            kk, lk = canon(k), self._canonical_lora_key(k)
            if kk in views:
                t = views[kk]
                if t.is_meta:
                    kind = self._matrix_kind(kk)
                    first = form.setdefault(kind, (v.dtype, kk))
                    if v.dtype != first[0]:
                        raise lib.QfxError(f"`{kk}` arrives as {v.dtype}, but `{first[1]}` of the same stacked kind {kind} arrived as "
                                           f"{first[0]}: the layers of a stacked kind must arrive in one format")
                    if tuple(v.shape) != tuple(t.shape):
                        raise lib.QfxError(f"`{kk}`: shape {tuple(v.shape)}, the model expects {tuple(t.shape)}")
                    o, n = t.storage_offset(), t.numel()
                    codes = fp8.as_e4m3(kk, v, self.dev)
                    self._fp8_store[kind].view(torch.uint8).view(-1)[o:o + n].copy_(codes.view(torch.uint8).reshape(-1))
                else:
                    t.copy_(v.to(self.dev, BF))
                seen.add(kk)
            elif lk in self._lora_params:
                self._lora_params[lk].copy_(v.to(self.dev, BF))
                seen.add(lk)
            else:
                unexpected.append(k)
        missing = [k for k in list(views) + list(self._lora_params) if k not in seen]
        if strict and (unexpected or [m for m in missing if "lora" not in m]):
            raise KeyError(f"load_state_dict: missing {missing[:5]}..., unexpected {unexpected[:5]}...")
        return missing, unexpected

    def _canonical_lora_key(self, k: str) -> str:
        """Spellings a LoRA tensor name arrives in -> this model's parameter name `<module>.lora_X.<adapter>.weight`:
        the PEFT state-dict form (identical), the diffusers LoRA-file form written by `save_lora`
        (`transformer.<module>.lora_X.weight`, base_trainer.py:858-875) and the adapter-less `get_peft_model_state_dict` form."""
        if ".lora_" not in k:
            return k
        if k.startswith("transformer."):
            k = k[len("transformer."):]
        head, _, tail = k.rpartition(".")
        if head.endswith(".lora_A") or head.endswith(".lora_B"):
            k = f"{head}.{self.adapter_name}.{tail}"
        return k

    def named_parameters(self, prefix="", recurse=True, remove_duplicate=True):
        for k, p in self._lora_params.items():
            yield (prefix + ("." if prefix else "") + k, p)

    def parameters(self, recurse=True):
        for _, p in self.named_parameters():
            yield p

    # ------------------------------------------------------------------------------------------------ LoRA registry
    def add_adapter(self, adapter_config, lora_alpha: float | None = None, target_modules=None, init_lora_weights=None,
                    seed: int = 0, b_std: float = 0.0, adapter_name: str = "default"):
        """`dit.add_adapter(LoraConfig(r=, lora_alpha=, init_lora_weights=, target_modules=), adapter_name=...)` exactly as the reference
        calls it (/root/reference/src/qflux/trainer/base_trainer.py:929-941) — `adapter_config` is any object with those attributes (a real
        `peft.LoraConfig` included; it is kept in `self.peft_config[adapter_name]` for `get_peft_model_state_dict`).  The short form
        `add_adapter(r, lora_alpha, target_modules=...)` is kept for scripts and tests.
        target_modules: list of name suffixes or one full regex (PEFT matching rules)."""
        if isinstance(adapter_config, int):
            r = adapter_config
            cfg = _LoraConfigLike(r=r, lora_alpha=lora_alpha if lora_alpha is not None else r,
                                  target_modules=list(DEFAULT_TARGETS) if target_modules is None else target_modules,
                                  init_lora_weights="gaussian" if init_lora_weights is None else init_lora_weights)
        else:
            cfg = adapter_config
            for attr, val in (("lora_dropout", 0.0), ("bias", "none"), ("use_dora", False), ("use_rslora", False)):
                if getattr(cfg, attr, val) not in (val, None):
                    raise NotImplementedError(f"LoraConfig.{attr}={getattr(cfg, attr)!r}: the fused path implements plain LoRA (dropout 0, no bias)")
            if getattr(cfg, "rank_pattern", None) or getattr(cfg, "alpha_pattern", None):
                raise NotImplementedError("per-module rank / alpha patterns are not supported by the fused path")
        check_rank(cfg.r)
        r, lora_alpha = int(cfg.r), float(cfg.lora_alpha)
        rp = padded_rank(r)
        target_modules = cfg.target_modules
        if isinstance(target_modules, (set, tuple)):
            target_modules = list(target_modules)
        init_lora_weights = cfg.init_lora_weights
        if init_lora_weights not in (True, "gaussian") and not (isinstance(init_lora_weights, str) and init_lora_weights.lower() == "gaussian"):
            raise NotImplementedError(f"init_lora_weights={init_lora_weights!r} (supported: True = kaiming-uniform A, 'gaussian')")
        init_lora_weights = "gaussian" if init_lora_weights is not True else True
        self.adapter_name = adapter_name
        self.peft_config = {adapter_name: cfg}
        self._hf_peft_config_loaded = True
        if self._lora_params:
            raise lib.QfxError("an adapter is already attached")
        table = dict(self._linear_table())
        D = self.D
        for full, (key, s_, d_in) in self._embed_table().items():
            table[full] = ((-1, key), (s_,), 0, d_in, D, 1)
        mod_table = self._mod_table()

        def match(full):
            if isinstance(target_modules, str):
                return re.fullmatch(target_modules, full) is not None
            return any(full == t or full.endswith("." + t) for t in target_modules)

        wanted = [full for full in table if match(full)]
        for k, v in self._weight_views().items():  # modules PEFT would adapt but the fused path cannot: fail loudly
            mod = k.rsplit(".", 1)[0]
            if k.endswith(".weight") and v.ndim == 2 and mod not in table and mod not in mod_table and match(mod):
                raise NotImplementedError(f"LoRA on `{mod}` is outside the fused hot path (SURVEY.md §8a a12)")
        wanted_mods = [full for full in mod_table if match(full)]
        if not wanted and not wanted_mods:
            raise lib.QfxError(f"no LoRA-capable module matches target_modules={target_modules!r}")
        self.lora_rank, self.lora_rp, self.lora_scaling = r, rp, float(lora_alpha) / r
        g = torch.Generator(device=self.dev).manual_seed(seed)
        off = 0
        for full in wanted:
            (l, grp), streams, slot, d_in, d_out, n_slots = table[full]
            site = self.sites.get((l, grp, streams[0]))
            if site is None:
                site = LoraSite(n_slots, d_in, d_out, rp, self.dev)
                for s in streams:
                    self.sites[(l, grp, s)] = site
            site.r = r
            A_view = site.A_pad[slot * rp: slot * rp + r]              # [r, in]  contiguous
            B_view = site.B_pad[slot * d_out:(slot + 1) * d_out, :r]   # [out, r] strided view
            if init_lora_weights == "gaussian":
                A_view.copy_(torch.randn(r, d_in, device=self.dev, generator=g) / r)
            else:
                A_view.copy_((torch.rand(r, d_in, device=self.dev, generator=g) * 2 - 1) / math.sqrt(d_in))
            if b_std > 0:
                B_view.copy_(torch.randn(d_out, r, device=self.dev, generator=g) * b_std)
            pA, pB = nn.Parameter(A_view), nn.Parameter(B_view)
            gA_off, gB_off = off, off + r * d_in
            off = gB_off + d_out * r
            site.members[slot] = (full, pA, pB, gA_off, gB_off, d_in, d_out)
            self._register_lora(full, pA, pB)
        # AdaLN modulation linears (M = batch rows only): factors stacked per kind so that forward and backward are a handful of
        # batched [B, .] products; gradients come from per-sample column reductions in the block backward (qfx_mod_grad)
        self._extra_members = []
        for kind in ("dbl", "sgl"):
            names = [f for f in wanted_mods if mod_table[f][0] == kind]
            if not names:
                continue
            n, C = len(names), mod_table[names[0]][2] * D
            A_all = torch.zeros(n, r, D, device=self.dev, dtype=BF)
            B_all = torch.zeros(n, C, r, device=self.dev, dtype=BF)
            if init_lora_weights == "gaussian":
                A_all.copy_(torch.randn(n, r, D, device=self.dev, generator=g) / r)
            else:
                A_all.copy_((torch.rand(n, r, D, device=self.dev, generator=g) * 2 - 1) / math.sqrt(D))
            if b_std > 0:
                B_all.copy_(torch.randn(n, C, r, device=self.dev, generator=g) * b_std)
            ga0, gb0 = off, off + n * r * D
            off = gb0 + n * C * r
            self.mod_sites[kind] = dict(idx=torch.tensor([mod_table[f][1] for f in names], device=self.dev),
                                        idx_list=[mod_table[f][1] for f in names], names=names, A=A_all,
                                        B=B_all, ga=ga0, gb=gb0, C=C, rows={mod_table[f][1] for f in names})
            for i, full in enumerate(names):
                pA, pB = nn.Parameter(A_all[i]), nn.Parameter(B_all[i])
                self._extra_members.append((full, pA, pB, ga0 + i * r * D, gb0 + i * C * r, D, C))
                self._register_lora(full, pA, pB)
        self.G32 = torch.zeros(off, device=self.dev, dtype=torch.float32)
        self.G16 = torch.zeros(off, device=self.dev, dtype=BF)
        self._gnorm_sq = torch.zeros(1, device=self.dev, dtype=torch.float32)
        self._gnorm_parts = torch.zeros(lib.DET_NORM_PARTIALS, device=self.dev, dtype=torch.float32)  # deterministic finalize
        self._gscratch = torch.zeros(5 * self.D * rp, device=self.dev, dtype=torch.float32)
        self._ws = self._ws_key = None  # per-block saved tensors depend on which sites exist
        self._train_ws, self._infer_ws = None, {}
        self._infer_graphs.clear()
        return self

    def _register_lora(self, full: str, pA: nn.Parameter, pB: nn.Parameter):
        """Publish the factors of module `full` under PEFT's names — in the flat name table AND as a real child-module path
        `<full>.lora_A.<adapter>` / `<full>.lora_B.<adapter>` so that module scans see them: `get_lora_layers(dit)` (what
        `accelerator_prepare` wraps / lists as FSDP `ignored_modules`, utils/lora_utils.py:25-38, base_trainer.py:340-342,383-387)."""
        a = self.adapter_name
        self._lora_params[f"{full}.lora_A.{a}.weight"] = pA
        self._lora_params[f"{full}.lora_B.{a}.weight"] = pB
        node = self
        for part in full.split("."):
            if part not in node._modules:
                node.add_module(part, nn.Module())
            node = node._modules[part]
        for which, p in (("lora_A", pA), ("lora_B", pB)):
            md = nn.ModuleDict()
            leaf = nn.Module()
            leaf.weight = p
            md[a] = leaf
            node.add_module(which, md)

    def set_adapter(self, adapter_name):
        """`transformer.set_adapter(adapter_name)` (base_trainer.py:941): one adapter is attached at a time."""
        names = [adapter_name] if isinstance(adapter_name, str) else list(adapter_name)
        if not self._lora_params or names != [self.adapter_name]:
            raise lib.QfxError(f"set_adapter({adapter_name!r}): attached adapter is {getattr(self, 'adapter_name', None)!r}")

    def active_adapters(self):
        return [self.adapter_name] if self._lora_params else []

    def cache_context(self, name: str):
        """diffusers `CacheMixin.cache_context` (a context manager that names the active branch for cache hooks): the reference's
        validation loop wraps every forward in it (qwen_image_edit_trainer.py:1236,1255).  No cache hooks here: a no-op context."""
        import contextlib
        return contextlib.nullcontext()

    @torch.no_grad()
    def merge_adapter(self, adapter_names=None):
        """PEFT `merge_adapter` (`BaseTrainer.merge_lora`, base_trainer.py:413-416): W <- W + scaling * B A for every adapted Linear, after
        which the adapter contributes nothing until `unmerge_adapter()`.  The factors are parked (the kernels always add the low-rank
        term, so a merged adapter is represented by lora_B = 0); the bf16 rounding of W + delta is PEFT's own."""
        if self._sharded is not None:
            raise lib.QfxError("merge_adapter: the frozen weights are sharded; merge on a replicated model")
        if self._nf4_kinds:
            raise lib.QfxError("merge_adapter: the frozen weights are NF4-resident (frozen_weights='nf4'); merge on a bf16 model")
        if self._fp8_kinds:
            raise lib.QfxError("merge_adapter: the frozen weights are FP8-resident (frozen_weights='fp8'): W + scaling * B A is not an "
                               "e4m3fn value; merge on a bf16 model")
        if not self._lora_params or getattr(self, "_merged", None):
            return
        views, parked = self._weight_views(), {}
        for k, pB in self._lora_params.items():
            if ".lora_B." not in k:
                continue
            mod = k.rsplit(".lora_B.", 1)[0]
            pA = self._lora_params[k.replace(".lora_B.", ".lora_A.")]
            W = views[mod + ".weight"]
            delta = (pB.float() @ pA.float()) * self.lora_scaling
            W.copy_((W.float() + delta).to(BF))
            parked[k] = pB.detach().clone()
            pB.zero_()
        self._merged = parked

    @torch.no_grad()
    def unmerge_adapter(self):
        """PEFT `unmerge_adapter`: subtract the merged delta again and restore lora_B."""
        parked = getattr(self, "_merged", None)
        if not parked:
            return
        views = self._weight_views()
        for k, B0 in parked.items():
            mod = k.rsplit(".lora_B.", 1)[0]
            pA = self._lora_params[k.replace(".lora_B.", ".lora_A.")]
            W = views[mod + ".weight"]
            W.copy_((W.float() - (B0.float() @ pA.float()) * self.lora_scaling).to(BF))
            self._lora_params[k].copy_(B0)
        self._merged = None

    def load_lora_adapter(self, pretrained_model_name_or_path_or_dict, prefix="transformer", adapter_name="default", **kwargs):
        """`transformer.load_lora_adapter(path, adapter_name=...)` (base_trainer.py:983): a diffusers-format LoRA file
        (`pytorch_lora_weights.safetensors`, keys `transformer.<module>.lora_A.weight`, what `save_lora` writes).  The rank is read from
        the tensors, alpha = rank (the format carries no alpha), targets = the modules present."""
        sd = pretrained_model_name_or_path_or_dict
        if not isinstance(sd, dict):
            import os
            import safetensors.torch
            path = sd if not os.path.isdir(sd) else os.path.join(sd, "pytorch_lora_weights.safetensors")
            sd = safetensors.torch.load_file(path)
        if prefix and any(k.startswith(prefix + ".") for k in sd):
            sd = {k[len(prefix) + 1:]: v for k, v in sd.items() if k.startswith(prefix + ".")}
        mods = sorted({k.rsplit(".lora_", 1)[0] for k in sd if ".lora_" in k})
        ranks = {v.shape[0] for k, v in sd.items() if ".lora_A" in k}
        if not mods or len(ranks) != 1:
            raise lib.QfxError(f"load_lora_adapter: expected LoRA tensors of one rank, found ranks {sorted(ranks)} in {len(sd)} tensors")
        r = ranks.pop()
        self.add_adapter(_LoraConfigLike(r=r, lora_alpha=r, target_modules="(" + "|".join(re.escape(m) for m in mods) + ")",
                                         init_lora_weights=True), adapter_name=adapter_name)
        missing, unexpected = self.load_state_dict(sd, strict=False)
        if unexpected or any("lora" in m for m in missing):
            raise lib.QfxError(f"load_lora_adapter: unexpected {unexpected[:3]}, missing {[m for m in missing if 'lora' in m][:3]}")

    def _unique_sites(self):
        seen = set()
        for site in self.sites.values():
            if id(site) not in seen:
                seen.add(id(site))
                yield site

    def _all_members(self):
        """(name, A param, B param, grad offset of A, grad offset of B, d_in, d_out) of every adapted Linear."""
        for site in self._unique_sites():
            yield from site.members.values()
        yield from getattr(self, "_extra_members", [])

    def bind_param_grads(self):
        """Point every LoRA `param.grad` at its slice of the flat bf16 gradient buffer (no copies)."""
        r = self.lora_rank
        for full, pA, pB, ga, gb, d_in, d_out in self._all_members():
            pA.grad = self.G16[ga: ga + r * d_in].view(r, d_in)
            pB.grad = self.G16[gb: gb + d_out * r].view(d_out, r)

    def lora_grad_views(self, flat=None):
        """{param name: view into a flat gradient buffer (default: the fp32 accumulator)}."""
        flat = self.G32 if flat is None else flat
        out, r = {}, self.lora_rank
        for full, pA, pB, ga, gb, d_in, d_out in self._all_members():
            out[f"{full}.lora_A.{self.adapter_name}.weight"] = flat[ga: ga + r * d_in].view(r, d_in)
            out[f"{full}.lora_B.{self.adapter_name}.weight"] = flat[gb: gb + d_out * r].view(d_out, r)
        return out

    # ------------------------------------------------------------------------------------------------ AdaLN-linear LoRA
    def _mods_view(self, ws, kind):
        C = self.mod_sites[kind]["C"]
        t = ws["mods"] if kind == "dbl" else ws["smods"]
        return t.view(t.shape[0], -1, C)

    def _mod_lora_fwd(self, ws, temb, kind_rows=None):
        """mods += scaling * lora_B(lora_A(silu(temb))) for every adapted modulation Linear, with PEFT's bf16 rounding points
        (lora_A output, lora_B output, the scaled product, the sum).  [B, .] operands: batched torch products, not a hot path.
        kind_rows = (kind, rows): only those rows (sharded weights produce the base modulation vectors block by block)."""
        if not self.mod_sites:
            return
        x = torch.nn.functional.silu(temb.float()).to(BF)  # the same rounded activation the modulation GEMV consumes
        ws["mod_x"] = x
        for kind, ms in self.mod_sites.items():
            sel = list(range(len(ms["names"])))
            if kind_rows is not None:
                sel = [i for i in sel if kind == kind_rows[0] and ms["idx_list"][i] in kind_rows[1]]
                if not sel:
                    continue
            if len(sel) == len(ms["names"]):  # everything (the un-sharded path): no list indexing -> no host-to-device index upload, which
                A, Bm, idx = ms["A"], ms["B"], ms["idx"]  # would be illegal inside the CUDA-graph capture of the step
            else:  # one block's rows (ringed weights): a device index made once per block, on the eager first step, so capture uploads nothing
                cache = ms.setdefault("sel_dev", {})
                if tuple(sel) not in cache:
                    cache[tuple(sel)] = torch.tensor(sel, device=self.dev)
                sel_t = cache[tuple(sel)]
                A, Bm, idx = ms["A"].index_select(0, sel_t), ms["B"].index_select(0, sel_t), ms["idx"].index_select(0, sel_t)
            t = torch.matmul(x.float()[None], A.float().transpose(1, 2)).to(BF)               # [n, B, r]
            d = torch.bmm(t.float(), Bm.float().transpose(1, 2)).to(BF)                       # [n, B, C]
            d = (d.float() * self.lora_scaling).to(BF)
            mv = self._mods_view(ws, kind)
            mv[:, idx] = (mv[:, idx].float() + d.float().permute(1, 0, 2)).to(BF)
            key = "mod_t_" + kind
            if key not in ws or ws[key].shape[1] != t.shape[1]:
                ws[key] = torch.zeros(len(ms["names"]), t.shape[1], t.shape[2], device=self.dev, dtype=BF)
            if len(sel) == len(ms["names"]):
                ws[key].copy_(t)
            else:
                ws[key].index_copy_(0, sel_t, t)

    def _mod_grad_buffers(self, ws):
        """fp32 accumulators for d mods (same layout as the modulation vectors), zeroed at the start of every backward."""
        for kind in self.mod_sites:
            key = "dmods" if kind == "dbl" else "dsmods"
            src = ws["mods"] if kind == "dbl" else ws["smods"]
            if key not in ws:
                ws[key] = torch.empty(src.shape, device=self.dev, dtype=torch.float32)
            ws[key].zero_()

    def _dmod(self, ws, kind, row, j):
        """fp32 [B, D] view: gradient of chunk j of modulation row `row` (None when that Linear has no adapter)."""
        ms = self.mod_sites.get(kind)
        if ms is None or row not in ms["rows"]:
            return None
        D = self.D
        t = ws["dmods" if kind == "dbl" else "dsmods"]
        off = row * ms["C"] + j * D
        return t[:, off: off + D]

    def _mod_lora_bwd(self, ws):
        """LoRA gradients of the modulation linears from the accumulated d mods:  dB = s * dmod^T t,  dA = s * (dmod B)^T x."""
        if not self.mod_sites:
            return
        r, D, x = self.lora_rank, self.D, ws["mod_x"].float()
        for kind, ms in self.mod_sites.items():
            n, C = len(ms["names"]), ms["C"]
            g = ws["dmods" if kind == "dbl" else "dsmods"]
            dm = g.view(g.shape[0], -1, C)[:, ms["idx"]].to(BF).float()                       # [B, n, C]  (autograd hands bf16 grads on)
            t = ws["mod_t_" + kind].float()                                                    # [n, B, r]
            u = (torch.bmm(dm.permute(1, 0, 2), ms["B"].float()) * self.lora_scaling).to(BF).float()   # [n, B, r]: the only real contraction (over C)
            # dB[n, c, r] = s * sum_b dm[b, n, c] t[n, b, r] and dA[n, r, d] = sum_b u[n, b, r] x[b, d] are rank-B updates (B = batch, 1-8):
            # as einsums cuBLAS ran them as K = B "GEMMs" at ~450 us per 6 sites (3.8 % of the FLUX config-3 step); as B fused
            # multiply-adds straight into the gradient accumulator they are one pass over it per sample
            GA = self.G32[ms["ga"]: ms["ga"] + n * r * D].view(n, r, D)
            GB = self.G32[ms["gb"]: ms["gb"] + n * C * r].view(n, C, r)
            if os.environ.get("QFX_MOD_EINSUM"):  # A/B switch: the einsum formulation
                GA.add_(torch.einsum("nbr,bd->nrd", u, x))
                GB.add_(torch.einsum("bnc,nbr->ncr", dm, t) * self.lora_scaling)
                continue
            for b in range(dm.shape[0]):
                GB.addcmul_(dm[b].unsqueeze(-1), t[:, b].unsqueeze(1), value=self.lora_scaling)
                GA.addcmul_(u[:, b].unsqueeze(-1), x[b].view(1, 1, D))

    def zero_lora_grads(self):
        self.G32.zero_()

    def finalize_grads(self, world_size: int = 1, max_norm: float = 0.0):
        """fp32 accumulator (already all-reduced by the caller) -> mean over ranks -> clip -> bf16 `param.grad`."""
        if torch.are_deterministic_algorithms_enabled():
            lib.grad_finalize_det(self.G32, 1.0 / world_size, max_norm, self._gnorm_sq, self.G16, scratch=self._gnorm_parts)
        else:
            lib.grad_finalize(self.G32, 1.0 / world_size, max_norm, self._gnorm_sq, self.G16)
        self.bind_param_grads()
        return self._gnorm_sq

    def close(self):
        """Teardown of a data-parallel run: unmap the memory this model maps from the other ranks (the deterministic gradient exchange's
        peer gradients, then the sharded frozen weights' peer shards).  Collective when either exists: every rank must call it.  G32
        moves back into an ordinary allocation; a model with sharded weights cannot run afterwards."""
        if self._grad_exchange:
            self._grad_exchange.close()
        self._grad_exchange = None
        for ring in (self._sharded, self._sharded_s):
            if ring is not None:
                ring.close()

    # ------------------------------------------------------------------------------------------------ helpers
    def _rows(self, ws, t, s):
        """rows of a stream-major [M, *] tensor: s=1 text, s=0 image."""
        return t[: ws["Mt"]] if s == 1 else t[ws["Mt"]:]

    def _rpb(self, ws, s):
        return ws["Limg"] if s == 0 else ws["T"]

    def _mod_grad(self, ws, g, rows_per_batch, **kw):
        """lib.mod_grad, or its fixed-order variant in a deterministic workspace."""
        if ws["det"]:
            lib.mod_grad_det(g, rows_per_batch, scratch=ws["det_scratch"], **kw)
        else:
            lib.mod_grad(g, rows_per_batch, **kw)

    def _plan_bands(self, ws, valid_img_rows):
        """Pad-to-max multi-resolution batch: the block GEMMs compute only the 256-row bands that hold valid image rows of a
        sample (lib.RowBands) and zero-fill the rest.  valid_img_rows: host list, one count per sample (None: dense batch).
        The tables are uploaded once per shape combination (never inside a captured step)."""
        ws["bands"] = None
        if valid_img_rows is None or os.environ.get("QFX_NO_RAGGED_GEMM"):
            return
        key = (tuple(int(v) for v in valid_img_rows), ws["Limg"])
        if key not in self._bands_cache:
            if len(self._bands_cache) >= 64:
                self._bands_cache.pop(next(iter(self._bands_cache)))
            plan = lib.RowBands.plan(key[0], ws["Limg"])
            self._bands_cache[key] = None if plan is None else lib.RowBands(plan[0], plan[1], self.dev)
        ws["bands"] = self._bands_cache[key]

    def _bands(self, ws, s):
        return ws.get("bands") if s == 0 else None

    # ------------------------------------------------------------------------------------------------ inference forward
    # A no-grad forward of 60 blocks is ~650 launches issued through ctypes: 40-65 ms of host time against 25 ms (B=1) to 95 ms (B=4) of
    # device time, and the validation sampler calls it 40 times per image (20 Euler steps x true CFG).  Like the training step, the second
    # forward of a given input signature is captured into a CUDA graph and later ones replay it (inputs copied into static buffers).
    def _infer(self, args):
        """`_forward_impl(*args, train=False)` -> prediction [B, Limg, C_out] (a view of workspace memory: callers clone it)."""
        return self._infer_graphs.run(self, lambda *a: self._forward_impl(*a, train=False), args, enabled=self.use_cuda_graph_inference)

    def _forward_tail(self, make_args):
        """The public `forward` once the family has turned its kwargs into `_forward_impl` arguments (`make_args()`): the fused
        autograd bridge when grad is enabled and an adapter is attached, the (graphed) no-grad forward otherwise."""
        if torch.is_inference_mode_enabled():
            # the reference's validation loop runs under torch.inference_mode() (qwen_image_edit_trainer.py:1219): workspaces and cached
            # tables allocated there would be inference tensors, which later no_grad / training calls may not update in place
            with torch.inference_mode(False), torch.no_grad():
                return self._forward_tail(make_args)
        args = make_args()
        if torch.is_grad_enabled() and self._lora_params:
            out = ModelFn.apply(self, args, *self._lora_params.values())
        else:
            out = self._infer(args).clone()
        kv = self._ws.get("kv_len")
        if kv is not None:  # padded image rows of a multi-resolution batch are returned as exact zeros (test_qwen_custom.py:672-692)
            valid = torch.arange(out.shape[1], device=out.device)[None, :] < (kv[:, None] - self._ws["T"])
            out = out * valid[..., None].to(out.dtype)
        return (out,)

    def _site(self, l, grp, s):
        return self.sites.get((l, grp, s))

    # one launch over both streams of a stream-major buffer (rows [0, Mt) text = stream 1, rows [Mt, M) image = stream 0);
    # `shift` / `scale` / `gate` are (image view, text view) pairs as returned by the mods(j) accessors
    def _ln_fwd2(self, ws, X, Y, shift, scale, mean=None, rstd=None):
        lib.ln_modulate_fwd_pair(X, Y, (shift[1], scale[1], ws["T"]), (shift[0], scale[0], ws["Limg"]), ws["Mt"], mean, rstd)

    def _ln_bwd2(self, ws, dy, x, mean, rstd, scale, dx, dres=None, gate=None, dx_gated=None):
        g = gate if gate else (None, None)
        lib.ln_modulate_bwd_pair(dy, x, mean, rstd, (scale[1], ws["T"], g[1]), (scale[0], ws["Limg"], g[0]), ws["Mt"], dx, dres=dres,
                                 dx_gated=dx_gated if gate else None)

    def _lora_T(self, ws, l, grp, s, X):
        """T = scaling * X @ A_pad^T  for the site (None if the site has no adapter)."""
        site = self._site(l, grp, s)
        if site is None:
            return None, None
        Tb = ws["loraT"][(l, grp, s)]
        lib.gemm([lib.gemm_problem(X, site.A_pad, Tb)], site.n * site.rp, X.shape[1], alpha=self.lora_scaling)
        return site, Tb

    def _lora_T_pair(self, ws, l, grp, src):
        """`_lora_T` for the image and the text stream of one weight group in ONE launch (two problems): these [M, Rp g] projections
        are latency-bound on 8-75 CTAs each, so running them side by side halves their cost.  Returns {s: (site, T)}."""
        res, probs = {}, []
        for s in (0, 1):
            site = self._site(l, grp, s)
            res[s] = (site, None if site is None else ws["loraT"][(l, grp, s)])
            if site is not None:
                probs.append((site.n * site.rp, lib.gemm_problem(self._rows(ws, src, s), site.A_pad, res[s][1])))
        K = src.shape[1]
        if len(probs) == 2 and probs[0][0] == probs[1][0]:
            lib.gemm([p for _, p in probs], probs[0][0], K, alpha=self.lora_scaling)
        else:
            for n, p in probs:
                lib.gemm([p], n, K, alpha=self.lora_scaling)
        return res

    def _embed_fwd(self, ws, key, s, X, dst):
        """Input embedder `key` (x_embedder / context_embedder / img_in / txt_in) with its optional fused LoRA pair."""
        W, b = self._wb(-1, key, s)
        site, Tb = self._lora_T(ws, -1, key, s, X)
        kw = dict(A2=Tb, B2=site.B_pad, kb2=site.rp // PAD) if site is not None else {}
        lib.gemm([lib.gemm_problem(X, W, dst, bias=b, **kw)], self.D, X.shape[1])
        ws["embed_in_" + key] = X

    def _embed_bwd(self, ws, key, s, dX0):
        """LoRA gradients of an input embedder from the gradient at the first block's input (the embedder input is data)."""
        if self._site(-1, key, s) is not None:
            self._lora_bwd(ws, -1, key, s, self._rows(ws, dX0, s), ws["embed_in_" + key], self.D)

    def _grouped(self, ws, l, grp, src, dst, N, K, epilogue, **epi):
        """One grouped GEMM over (image, text) rows of block l for weight group `grp` with optional fused LoRA."""
        probs = []
        lora = self._lora_T_pair(ws, l, grp, src)
        for s in (0, 1):
            A = self._rows(ws, src, s)
            site, Tb = lora[s]
            kw = {}
            if site is not None:
                kw = dict(A2=Tb, B2=site.B_pad, kb2=site.rp // PAD)
            for k, v in epi.items():
                if v is None:
                    continue
                if k == "gate":
                    kw["gate"], kw["rows_per_batch"] = v[s], self._rpb(ws, s)
                else:
                    kw[k] = self._rows(ws, v, s)
            W, b = self._wb(l, grp, s)
            probs.append(lib.gemm_problem(A, W, self._rows(ws, dst, s), bias=b, row_bands=self._bands(ws, s), **kw))
        fused3 = any(p.kb2 for p in probs) and self._site_n(l, grp) == 3
        lib.gemm(probs, N, K, epilogue=epilogue, lora_group_n=(N // 3 if fused3 else 0))

    def _site_n(self, l, grp):
        for s in (0, 1):
            site = self._site(l, grp, s)
            if site is not None:
                return site.n
        return 0

    def _lora_U_problems(self, ws, l, grp, s, dY, n_out_each):
        """GEMM problems of U_g = scaling * dY_g . B_g for the slots g of one site (U feeds the fused dgrad and dA)."""
        site = self._site(l, grp, s)
        rp = site.rp
        U = self._rows(ws, ws["U"], s)[:, : site.n * rp]
        return [lib.gemm_problem(dY[:, g * n_out_each:(g + 1) * n_out_each], site.B_pad[g * n_out_each:(g + 1) * n_out_each],
                                 U[:, g * rp:(g + 1) * rp]) for g in range(site.n)]

    def _lora_wgrads(self, ws, l, grp, s, dY, Xsaved, n_out_each):
        """Weight gradients of one site on the tensor cores: dB_g[out, r] += dY_g^T T_g (grouped-diagonal), dA_g[r, in] += U_g^T X."""
        site = self._site(l, grp, s)
        r, rp, Tb = site.r, site.rp, ws["loraT"][(l, grp, s)]
        U = self._rows(ws, ws["U"], s)[:, : site.n * rp]
        gB, gA = [], []
        for g in range(site.n):
            if g in site.members:
                full, pA, pB, ga, gb, d_in, d_out = site.members[g]
                gB.append(self.G32[gb:])
                gA.append(self.G32[ga:])
            else:  # slot without an adapter (e.g. LoRA on to_q/to_v only): its zero factors produce zeros -> scratch
                gB.append(self._gscratch)
                gA.append(self._gscratch)
        det = {"scratch": ws["det_scratch"]} if ws["det"] else {}
        wgrad_tc = lib.lora_wgrad_tc_det if det else lib.lora_wgrad_tc
        wgrad_tc(dY, Tb, gB, r, 1, r, mode=1 if site.n > 1 else 0, Dg=n_out_each if site.n > 1 else 0, **det)
        if Xsaved.shape[1] % 128 == 0:
            wgrad_tc(Xsaved, U, gA, 1, Xsaved.shape[1], r, mode=0, **det)
        else:  # 64-channel latent embedder: too narrow for the wgmma tile, a [r, 64] result on the CUDA cores, in rank chunks of
            # the widths that kernel takes (disjoint columns of U and rows of dA)
            d_in = Xsaved.shape[1]
            for g in range(site.n):
                for c0, w in rank_chunks(r):
                    (lib.lora_wgrad_det if det else lib.lora_wgrad)(Xsaved, U[:, g * rp + c0:(g + 1) * rp], gA[g][c0 * d_in:], 1, d_in, w, **det)
        return U, site.A_pad, site.n * rp // PAD

    def _lora_bwd(self, ws, l, grp, s, dY, Xsaved, n_out_each):
        """LoRA part of a linear's backward for one site: U = s*dY.B (for the fused dgrad) and the weight gradients.
        dY [M_s, n_slots*out]; Xsaved [M_s, in] is the linear's input (for dA)."""
        if self._site(l, grp, s) is None:
            return None
        lib.gemm(self._lora_U_problems(ws, l, grp, s, dY, n_out_each), self.lora_rp, n_out_each, trans_b=True, alpha=self.lora_scaling)
        return self._lora_wgrads(ws, l, grp, s, dY, Xsaved, n_out_each)

    def _lora_bwd_pair(self, ws, l, grp, dY, Xsaved, n_out_each):
        """`_lora_bwd` for both streams of a weight group with ALL their U projections (up to 3 slots x 2 streams) in one launch.
        dY / Xsaved are stream-major [M, .] buffers.  Returns {s: (U, A_pad, kb2 = n Rp / 64) | None}."""
        probs = []
        for s in (0, 1):
            if self._site(l, grp, s) is not None:
                probs += self._lora_U_problems(ws, l, grp, s, self._rows(ws, dY, s), n_out_each)
        if probs:
            lib.gemm(probs, self.lora_rp, n_out_each, trans_b=True, alpha=self.lora_scaling)
        return {s: (self._lora_wgrads(ws, l, grp, s, self._rows(ws, dY, s), self._rows(ws, Xsaved, s), n_out_each)
                    if self._site(l, grp, s) is not None else None) for s in (0, 1)}

    def _dgrad_grouped(self, ws, l, grp, dY, dXout, N, K, n_out_each, Xsaved, epilogue=lib.EPI_BIAS, aux=None, resid=None):
        """dX = dY . W (+ U . A) for both streams of weight group `grp` (W stored [out, in] = [K_red, N])."""
        probs = []
        if Xsaved is None:
            assert self._site(l, grp, 0) is None and self._site(l, grp, 1) is None, "a LoRA site needs the saved input of its linear"
        lbs = self._lora_bwd_pair(ws, l, grp, dY, Xsaved, n_out_each) if Xsaved is not None else {0: None, 1: None}
        for s in (0, 1):
            dYs = self._rows(ws, dY, s)
            lb = lbs[s]
            kw = {}
            if lb is not None:
                kw = dict(A2=lb[0], B2=lb[1], kb2=lb[2])
            if aux is not None:
                kw["aux"] = self._rows(ws, aux, s)
            if resid is not None:
                kw["resid"] = self._rows(ws, resid, s)
            probs.append(lib.gemm_problem(dYs, self._wb(l, grp, s)[0], self._rows(ws, dXout, s), row_bands=self._bands(ws, s), **kw))
        lib.gemm(probs, N, K, trans_b=True, epilogue=epilogue)

    def _dgrad_attn_out(self, ws, probs_in, O, N, K):
        """Out-projection dgrad whose epilogue hands the result straight to the attention backward (EPI_ATTN_DO): dO goes head-major
        into ws['dOj'] and delta = rowsum(dO * O) into ws['delta'] — no token-major dO, no separate attn_delta pass.
        probs_in: per stream (dY rows, W, lora kw).  Runs dense (no row bands): every (b, s) of dOj / delta must be defined."""
        T, Limg = ws["T"], ws["Limg"]
        if os.environ.get("QFX_NO_FUSED_DO"):  # A/B switch: the round-1 sequence (token-major dO, then the attn_delta pass)
            if "dO" not in ws:
                ws["dO"] = torch.empty(ws["Mt"] + ws["Mi"], N, device=self.dev, dtype=BF)
            lib.gemm([lib.gemm_problem(dYs, W, self._rows(ws, ws["dO"], s), **kw) for s, (dYs, W, kw) in enumerate(probs_in)], N, K, trans_b=True)
            lib.attn_delta_pair(O, ws["dO"], ws["delta"], (T, 0), (Limg, T), ws["Mt"], ws["dOj"])
            return
        probs = []
        for s, (dYs, W, kw) in enumerate(probs_in):
            probs.append(lib.gemm_problem(dYs, W, ws["dOj"], aux=self._rows(ws, O, s), delta=ws["delta"], rows_per_batch=self._rpb(ws, s),
                                          s_offset=T if s == 0 else 0, **kw))
        lib.gemm(probs, N, K, trans_b=True, epilogue=lib.EPI_ATTN_DO)

    # ------------------------------------------------------------------------------------------------ double-stream block
    # mods(j): j-th D-wide chunk (shift1, scale1, gate1, shift2, scale2, gate2) -> (img view, txt view), each [B, D]
    def _double_fwd(self, ws, l, Xin, Xout, save, mods, recompute=False):
        """recompute: regenerate the saved tensors of block l for its backward.  The down projection is skipped then (its output,
        the next block's input, is kept) unless its un-gated output feeds an AdaLN-LoRA gate gradient; it then rewrites Xout,
        which no later step of the backward reads."""
        D = self.D
        T, Limg, Mt = ws["T"], ws["Limg"], ws["Mt"]
        st, qkv, O, xmid, u = save["stats"], save["qkv"], save["O"], save["xmid"], save["u"]
        w = self.w
        xm1 = save.get("xm1", ws["xm"])  # kept per block in training: it is the LoRA input of the q|k|v sites in the backward
        Qs, Ks, Vs = save.get("Q", ws["Q"]), save.get("K", ws["K"]), save.get("V", ws["V"])
        # stream-major rows: text (stream 1) first, image (stream 0) behind it -> ONE launch per op covers both streams
        lib.ln_modulate_fwd_pair(Xin, xm1, (mods(0)[1], mods(1)[1], T), (mods(0)[0], mods(1)[0], Limg), Mt, st[0], st[1])
        self._grouped(ws, l, "qkv", xm1, qkv, 3 * D, D, lib.EPI_BIAS)
        qn = w["qknorm_w"][l]
        lib.qk_norm_rope_fwd_pair(qkv, (qn[2], qn[3], T, 0), (qn[0], qn[1], Limg, T), Mt, ws["rope"], Qs, Ks, Vs, round_mid=self.round_mid)
        lib.attn_fwd(Qs, Ks, Vs, O[:Mt], O[Mt:], T, save["lse"], kv_len=ws.get("kv_len"), txt_len=ws.get("txt_len"))
        self._grouped(ws, l, "out", O, xmid, D, D, lib.EPI_RESID_GATE, resid=Xin, gate=mods(2), out2=save.get("y_attn"))
        lib.ln_modulate_fwd_pair(xmid, ws["xm"], (mods(3)[1], mods(4)[1], T), (mods(3)[0], mods(4)[0], Limg), Mt, st[2], st[3])
        h = save.get("h", ws["h"])  # kept per block only when ff.net.2 carries LoRA (its input is needed for dA)
        self._grouped(ws, l, "up", ws["xm"], h, 4 * D, D, lib.EPI_GELU, out2=u)
        if not recompute or self._keeps_gate_out(l):
            self._grouped(ws, l, "down", h, Xout, D, 4 * D, lib.EPI_RESID_GATE, resid=xmid, gate=mods(5), out2=save.get("y_mlp"))

    def _attn_bwd_core(self, ws, qkv, O, lse, wq_wk, save=None):
        """dO (head-major ws['dOj'] + ws['delta'], written by the out-projection dgrad: _dgrad_attn_out) -> dqkv (ws['dqkv']);
        wq_wk(s) -> (wq, wk) norm weights of stream s.
        The normalised / rotated Q, K, V come from the block's saved tensors when present, else they are regenerated."""
        T, Limg, Mt = ws["T"], ws["Limg"], ws["Mt"]
        have = save is not None and "Q" in save
        Qs, Ks, Vs = (save["Q"], save["K"], save["V"]) if have else (ws["Q"], ws["K"], ws["V"])
        g_txt, g_img = (*wq_wk(1), T, 0), (*wq_wk(0), Limg, T)  # (wq, wk, tokens per sample, joint offset) of the two row groups
        if not have:
            lib.qk_norm_rope_fwd_pair(qkv, g_txt, g_img, Mt, ws["rope"], Qs, Ks, Vs, round_mid=self.round_mid)
        # dQ (fp32, 118 MB at the benchmark shape) is zero-filled right before the kernel that reduces into it.  Letting the consumer
        # below re-zero what it reads (QFX_DQ_CLEAR_IN_CONSUMER=1) removes the fill but makes the step 5 % SLOWER (same box: 344.7 vs
        # 326.4 ms): the red.global.add traffic then lands on lines that left L2 a whole block earlier.
        consumer_clears = bool(os.environ.get("QFX_DQ_CLEAR_IN_CONSUMER"))
        if not (consumer_clears and ws.get("dQ_clean")):
            ws["dQ"].zero_()
        ws["dQ_clean"] = False
        (lib.attn_bwd_det if ws["det"] else lib.attn_bwd)(Qs, Ks, Vs, ws["dOj"], lse, ws["delta"], ws["dQ"], ws["dK"], ws["dV"],
                                                          kv_len=ws.get("kv_len"), txt_len=ws.get("txt_len"), split=T)
        lib.qk_norm_rope_bwd_pair(ws["dQ"], ws["dK"], ws["dV"], qkv, g_txt, g_img, Mt, ws["rope"], ws["dqkv"], round_mid=self.round_mid,
                                  clear_dq=consumer_clears)
        ws["dQ_clean"] = consumer_clears

    def _double_bwd(self, ws, l, Xin, dX, dXn, save, mods, prev_gate):
        """dX: grad wrt the block output (ws['dY'] already holds dX * gate2).  Writes the grad wrt the block input to dXn
        and, when prev_gate is given, dXn * prev_gate to ws['dY'] for the block before."""
        D = self.D
        st, qkv, O, xmid, u = save["stats"], save["qkv"], save["O"], save["xmid"], save["u"]
        w = self.w
        dm = lambda s, j: self._dmod(ws, "dbl", 2 * l + s, j)  # fp32 [B, D] accumulators of d(shift1, scale1, gate1, shift2, scale2, gate2)
        for s in (0, 1):
            if dm(s, 5) is not None:  # d gate2 = sum_t dXout * mlp_out  (before dX is overwritten with dXmid below)
                self._mod_grad(ws, self._rows(ws, dX, s), self._rpb(ws, s), m=self._rows(ws, save["y_mlp"], s), prod_out=dm(s, 5))
        # ---- MLP branch
        self._dgrad_grouped(ws, l, "down", ws["dY"], ws["dbig"], 4 * D, D, D, save.get("h"), epilogue=lib.EPI_DGELU, aux=u)
        if self._site(l, "up", 0) or self._site(l, "up", 1):  # LoRA input = xm2, recomputed from the statistics
            self._ln_fwd2(ws, xmid, ws["xm"], mods(3), mods(4))
        self._dgrad_grouped(ws, l, "up", ws["dbig"], ws["dxm"], D, 4 * D, 4 * D, ws["xm"])
        # ---- norm2 backward: dXmid = dX + LN_bwd ; also emit dXmid * gate1 for the attention out-projection
        for s in (0, 1):
            if dm(s, 3) is not None:  # d shift2 = sum_t dy ; d scale2 = sum_t dy * LN(xmid)
                self._mod_grad(ws, self._rows(ws, ws["dxm"], s), self._rpb(ws, s), sum_out=dm(s, 3), m=self._rows(ws, xmid, s),
                               prod_out=dm(s, 4), mean=self._rows(ws, st[2], s), rstd=self._rows(ws, st[3], s))
        T, Limg, Mt = ws["T"], ws["Limg"], ws["Mt"]
        lib.ln_modulate_bwd_pair(ws["dxm"], xmid, st[2], st[3], (mods(4)[1], T, mods(2)[1]), (mods(4)[0], Limg, mods(2)[0]), Mt, dX,
                                 dres=dX, dx_gated=ws["dY"])
        for s in (0, 1):
            if dm(s, 2) is not None:  # d gate1 = sum_t dXmid * attn_out   (dX holds dXmid now)
                self._mod_grad(ws, self._rows(ws, dX, s), self._rpb(ws, s), m=self._rows(ws, save["y_attn"], s), prod_out=dm(s, 2))
        # ---- attention output projection (LoRA input = O), attention, q|k|v projection (LoRA input = xm1, recomputed)
        lbs = self._lora_bwd_pair(ws, l, "out", ws["dY"], O, D)
        self._dgrad_attn_out(ws, [(self._rows(ws, ws["dY"], s), self._wb(l, "out", s)[0],
                                   dict(A2=lbs[s][0], B2=lbs[s][1], kb2=lbs[s][2]) if lbs[s] is not None else {}) for s in (0, 1)], O, D, D)
        self._attn_bwd_core(ws, qkv, O, save["lse"], lambda s: (w["qknorm_w"][l, 2 * s], w["qknorm_w"][l, 2 * s + 1]), save)
        xm1 = save.get("xm1")
        if xm1 is None:
            xm1 = ws["xm"]
            if self._site(l, "qkv", 0) or self._site(l, "qkv", 1):
                self._ln_fwd2(ws, Xin, xm1, mods(0), mods(1))
        self._dgrad_grouped(ws, l, "qkv", ws["dqkv"], ws["dxm"], D, 3 * D, D, xm1)
        # ---- norm1 backward: dXin = dXmid + LN_bwd ; emit dXin * (gate of the block before)
        for s in (0, 1):
            if dm(s, 0) is not None:
                self._mod_grad(ws, self._rows(ws, ws["dxm"], s), self._rpb(ws, s), sum_out=dm(s, 0), m=self._rows(ws, Xin, s),
                               prod_out=dm(s, 1), mean=self._rows(ws, st[0], s), rstd=self._rows(ws, st[1], s))
        pg = prev_gate if prev_gate else (None, None)
        lib.ln_modulate_bwd_pair(ws["dxm"], Xin, st[0], st[1], (mods(1)[1], T, pg[1]), (mods(1)[0], Limg, pg[0]), Mt, dXn, dres=dX,
                                 dx_gated=ws["dY"] if prev_gate else None)

    # ------------------------------------------------------------------------------------------------ block stack and output head
    def _mods(self, ws, l):
        """j -> (image view, text view) of the j-th D-wide modulation chunk of double block l (shift1,scale1,gate1,shift2,scale2,gate2)."""
        D = self.D

        def f(j):
            return tuple(ws["mods"][:, ((l * 2 + s) * 6 + j) * D: ((l * 2 + s) * 6 + j + 1) * D] for s in (0, 1))
        return f

    def _smod(self, ws, l, j):
        """j-th chunk (shift, scale, gate) of single block l — the same [B, D] vector for both row groups."""
        D = self.D
        v = ws["smods"][:, (l * 3 + j) * D: (l * 3 + j + 1) * D]
        return (v, v)

    def _last_gate(self, ws, blk):
        """gate multiplying the residual branch that ENDS block `blk` (global index over double then single blocks)."""
        return self._mods(ws, blk)(5) if blk < self.L else self._smod(ws, blk - self.L, 2)

    def _blocks_and_head_fwd(self, ws, train):
        """Every block (double blocks, then single blocks) from the embedded tokens in ws["X"][0], then the output head on the image
        rows: AdaLayerNormContinuous (scale, shift) + proj_out.  Returns the prediction [B, Limg, C_out] (workspace memory)."""
        D, L, Mt, w, sh = self.D, self.L, ws["Mt"], self.w, self._blk_rings
        nb = L + self.Ls
        xi = lambda i: ws["X"][i] if train else ws["X"][i & 1]
        for ring in self._expand_rings or ():  # every forward fills the same blocks: eager, captured and replayed alike
            if ring is not None:
                ring.reset()
        for blk in range(nb):
            if sh is not None:  # block blk's weights arrive through its ring (block blk+1's fill starts now, on the side stream)
                self._acquire(blk, blk + 1)
                self._block_mods(ws, blk)
            if blk < L:
                self._double_fwd(ws, blk, xi(blk), xi(blk + 1), ws["dbl"][blk if train else 0], self._mods(ws, blk))
            else:
                self._single_fwd(ws, blk - L, xi(blk), xi(blk + 1), ws["sgl"][(blk - L) if train else 0])
            if sh is not None:
                self._release(blk)
        self._join_expand_rings()
        Xl = ws["Xlast"] = xi(nb)
        lib.ln_modulate_fwd(Xl[Mt:], ws["hn"], ws["fmod"][:, D:], ws["fmod"][:, :D], ws["Limg"], ws["fstats"][0], ws["fstats"][1])
        lib.gemm([lib.gemm_problem(ws["hn"], w["proj_out_w"], ws["pred"], bias=w["proj_out_b"])], self.C_out, D)
        return ws["pred"].view(ws["B"], ws["Limg"], self.C_out)

    def _backward_impl(self, dpred):
        """dpred: [B*Limg, C_out] bf16 gradient of the loss wrt the prediction; accumulates LoRA grads into self.G32."""
        ws = self._ws
        assert ws is not None and self._ws_key[3], "backward needs a training-mode forward first"
        Limg, Mt = ws["Limg"], ws["Mt"]
        D, L, w = self.D, self.L, self.w
        nb = L + self.Ls
        self._mod_grad_buffers(ws)
        # --- head: proj_out dgrad -> final AdaLN backward.  Text rows of the last block output receive no gradient.
        lib.gemm([lib.gemm_problem(dpred, w["proj_out_w"], ws["dhn"])], D, self.C_out, trans_b=True)
        dX = ws["dX"][nb & 1]
        dX[:Mt].zero_()
        ws["dY"][:Mt].zero_()
        lib.ln_modulate_bwd(ws["dhn"], ws["Xlast"][Mt:], ws["fstats"][0], ws["fstats"][1], ws["fmod"][:, :D], Limg, dX[Mt:],
                            gate=self._last_gate(ws, nb - 1)[0], dx_gated=ws["dY"][Mt:])
        for blk in range(nb - 1, -1, -1):
            dXn = ws["dX"][blk & 1]
            prev = self._last_gate(ws, blk - 1) if blk > 0 else None
            if self._blk_rings is not None:
                self._acquire(blk, blk - 1)
            if blk in ws["plan"].recompute:  # regenerate the block's saved tensors into the scratch dict (its weights are resident now)
                if blk < L:
                    self._double_fwd(ws, blk, ws["X"][blk], ws["X"][blk + 1], ws["dbl"][blk], self._mods(ws, blk), recompute=True)
                else:
                    self._single_fwd(ws, blk - L, ws["X"][blk], ws["X"][blk + 1], ws["sgl"][blk - L], recompute=True)
            if blk < L:
                self._double_bwd(ws, blk, ws["X"][blk], dX, dXn, ws["dbl"][blk], self._mods(ws, blk), prev)
            else:
                self._single_bwd(ws, blk - L, ws["X"][blk], dX, dXn, ws["sgl"][blk - L], prev)
            if self._blk_rings is not None:
                self._release(blk)
            dX = dXn
        self._join_expand_rings()
        self._mod_lora_bwd(ws)
        for key, s, _ in self._embed_table().values():
            self._embed_bwd(ws, key, s, dX)

    # ------------------------------------------------------------------------------------------------ workspace pieces
    def _keeps_gate_out(self, l, kind="dbl"):
        """Block l's un-gated branch outputs are saved: an AdaLN linear of the block carries LoRA (they feed d gate)."""
        rows = self.mod_sites.get(kind, {}).get("rows", ())
        return (2 * l in rows or 2 * l + 1 in rows) if kind == "dbl" else l in rows

    def _saved_entries(self, kind, blocks, B, S, train):
        """[(group, name, shape, dtype)] of the saved dict serving `blocks` (indices of one block kind; every optional entry any of
        them needs).  Allocation runs group by group over the dicts of a kind."""
        D, H, M, f32 = self.D, self.H, B * S, torch.float32
        if kind == "dbl":
            ent = [(0, "stats", (4, M), f32), (0, "qkv", (M, 3 * D), BF), (0, "O", (M, D), BF), (0, "lse", (B, H, S), f32),
                   (0, "xmid", (M, D), BF), (0, "u", (M, 4 * D), BF)]
            if train and self.keep_qkv:  # +4 x [M, D] per block in HBM instead of regenerating them in the backward
                ent += [(1, "Q", (B, H, S, 128), BF), (1, "K", (B, H, S, 128), BF), (1, "V", (B, H, S, 128), BF), (1, "xm1", (M, D), BF)]
            if train and any(self._site(l, "down", 0) or self._site(l, "down", 1) for l in blocks):
                ent.append((2, "h", (M, 4 * D), BF))  # the LoRA input of ff.net.2
            if train and any(self._keeps_gate_out(l) for l in blocks):  # un-gated branch outputs, needed for d gate
                ent += [(2, "y_attn", (M, D), BF), (2, "y_mlp", (M, D), BF)]
            return ent
        # single blocks keep cat[attn | gelu(mlp)] — the input of proj_out — in ONE [M, 5D] buffer: attention and the GELU epilogue
        # write straight into its column ranges (no concat), proj_out is a plain K = 5D contraction, and the buffer is the LoRA
        # input of proj_out in the backward
        ent = [(0, "stats", (2, M), f32), (0, "qkv", (M, 3 * D), BF), (0, "cat", (M, 5 * D), BF), (0, "lse", (B, H, S), f32),
               (0, "u", (M, 4 * D), BF)]
        if train and any(self._keeps_gate_out(l, "sgl") for l in blocks):
            ent.append((1, "y_out", (M, D), BF))
        return ent

    def _det_scratch_floats(self, B, T, Limg):
        """fp32 scratch of the deterministic reductions of one training step: the largest need over the loss, every modulation-gradient
        row group and every LoRA site's weight gradients (lib.det_scratch_* restate qfx.h's rules)."""
        S = T + Limg
        n = lib.DET_LOSS_PARTIALS
        for M, rpb in ((B * Limg, Limg), (B * T, T), (B * S, S)):
            n = max(n, lib.det_scratch_mod_grad(M, rpb, self.D))
        for site in self.sites.values():
            d_in, d_out = site.A_pad.shape[1], site.B_pad.shape[0] // site.n
            for M in (B * Limg, B * T, B * S):
                n = max(n, lib.det_scratch_wgrad_tc(M, site.n * d_out, 1, site.r))
                n = max(n, lib.det_scratch_wgrad_tc(M, d_in, site.n, site.r) if d_in % 128 == 0 else
                        max(lib.det_scratch_wgrad(M, d_in, w) for _, w in rank_chunks(site.r)))
        return n

    def _fixed_entries(self, B, T, Limg, train, nblk, extra, det=False):
        """([(name, shape, dtype)] allocated before the saved dicts, [...] after them): every workspace buffer whose size does
        not depend on the activation plan.  `extra`: the family's conditioning buffers [(name, shape)] (bf16), allocated last.
        det: the step runs the deterministic kernels, whose reduction scratch is one more fixed buffer."""
        D, H, S, Mi, f32 = self.D, self.H, T + Limg, B * Limg, torch.float32
        M = B * S
        pre = [("X", (nblk + 1 if train else 2, M, D), BF), ("xm", (M, D), BF), ("h", (M, 4 * D), BF),
               ("Q", (B, H, S, 128), BF), ("K", (B, H, S, 128), BF), ("V", (B, H, S, 128), BF)]
        post = [("hn", (Mi, D), BF), ("pred", (Mi, self.C_out), BF), ("fstats", (2, Mi), f32)]
        post += [(("loraT", key), (Mi if key[2] == 0 else B * T, site.n * site.rp), BF) for key, site in self.sites.items()]
        if train:
            post += [("dX", (2, M, D), BF), ("dY", (M, D), BF), ("dbig", (M, 4 * D), BF), ("dqkv", (M, 3 * D), BF), ("dxm", (M, D), BF),
                     ("dOj", (B, H, S, 128), BF), ("dK", (B, H, S, 128), BF), ("dV", (B, H, S, 128), BF), ("dQ", (B, H, S, 128), f32),
                     ("delta", (B, H, S), f32), ("U", (M, 3 * self.lora_rp), BF), ("dhn", (Mi, D), BF), ("dpred", (Mi, self.C_out), BF),
                     ("loss", (1,), f32)]
            if det:
                post.append(("det_scratch", (self._det_scratch_floats(B, T, Limg),), f32))
        return pre, post + [(k, s, BF) for k, s in extra]

    def _activation_limit_now(self):
        if self._activation_limit is not None:
            return self._activation_limit
        if self.dev.type != "cuda":  # host-only models: nothing to plan against
            return None
        return torch.cuda.mem_get_info(self.dev)[0] - ACTIVATION_HEADROOM

    def _alloc_common(self, ws, B, T, Limg, train, n_double, n_single=0, extra=(), det=False):
        """The workspace of one (B, T, Limg, train) shape.  Training: every block either keeps its own saved dict or, when the
        activation plan recomputes it, points at the one scratch dict of its kind (plan_activation_memory; planned before
        anything is allocated)."""
        D = self.D
        Mt, Mi = B * T, B * Limg
        M, S = Mt + Mi, T + Limg
        nbytes = lambda shape, dt: math.prod(shape) * dt.itemsize
        ws.update(B=B, T=T, Limg=Limg, S=S, Mt=Mt, Mi=Mi, M=M, det=det)
        nblk = n_double + n_single
        nd = n_double if train else min(1, n_double)
        ns = n_single if train else min(1, n_single)
        pre, post = self._fixed_entries(B, T, Limg, train, nblk, extra, det)
        kinds = [("dbl", l) for l in range(nd)] + [("sgl", l) for l in range(ns)]
        plan = ActivationPlan((), 0, 0, 0, None)
        if train:
            per_block = [(k, {n: nbytes(s, dt) for _, n, s, dt in self._saved_entries(k, (l,), B, S, True)}) for k, l in kinds]
            plan = plan_activation_memory(per_block, sum(nbytes(s, dt) for _, s, dt in pre + post), self._activation_limit_now())
        ws["plan"] = plan
        for name, shape, dt in pre:
            ws[name] = torch.empty(shape, device=self.dev, dtype=dt)
        for kind, n in (("dbl", nd), ("sgl", ns)):
            first = n_double if kind == "sgl" else 0  # global index of the kind's block 0
            rec = [l for l in range(n) if first + l in plan.recompute]
            slots = [([l], {}) for l in range(n) if first + l not in plan.recompute] + ([(rec, {})] if rec else [])
            ents = [(d, self._saved_entries(kind, ls, B, S, train)) for ls, d in slots]
            for g in (0, 1, 2):
                for d, ent in ents:
                    for grp, name, shape, dt in ent:
                        if grp == g:
                            d[name] = torch.empty(shape, device=self.dev, dtype=dt)
            ws[kind] = [next(d for ls, d in slots if l in ls) for l in range(n)]
        for blk in ws["sgl"]:
            blk["O"], blk["h"] = blk["cat"][:, :D], blk["cat"][:, D:]
        ws["loraT"] = {}
        for name, shape, dt in post:
            if isinstance(name, tuple):
                ws["loraT"][name[1]] = torch.zeros(shape, device=self.dev, dtype=dt)
            elif name == "loss":
                ws["loss"] = torch.zeros(shape, device=self.dev, dtype=dt)
            else:
                ws[name] = torch.empty(shape, device=self.dev, dtype=dt)
        return ws

    def _get_workspace(self, key, build):
        """key = (B, T, Limg, train, det), det: torch.are_deterministic_algorithms_enabled() of a training forward.  One training workspace (tens of GB of saved activations) and up to three inference workspaces
        (a few hundred MB each: validation alternates between the prompt and the negative prompt, whose text lengths may differ) stay
        allocated, so switching between them neither re-allocates nor invalidates the CUDA graphs captured on them."""
        if self._ws_key == key:
            return self._ws
        train = bool(key[3])
        cached = self._train_ws if train else self._infer_ws.get(key)
        if cached is not None and (not train or cached[0] == key):
            ws = cached[1] if train else cached
        else:
            if train:
                self._ws = self._train_ws = None  # a new training shape: the old saved activations go first
                if torch.cuda.is_available():
                    torch.cuda.empty_cache()
            ws = build()
            if train:
                self._train_ws = (key, ws)
            else:
                if len(self._infer_ws) >= 3:
                    self._infer_ws.pop(next(iter(self._infer_ws)))
                self._infer_ws[key] = ws
        self._ws, self._ws_key = ws, key
        return ws

    def _activate_ws(self, ws, key) -> bool:
        """Make a workspace a captured graph was recorded on current again; False if the model no longer holds it."""
        held = (self._train_ws is not None and self._train_ws[1] is ws) or any(w is ws for w in self._infer_ws.values())
        if held:
            self._ws, self._ws_key = ws, key
        return held


class GraphCache:
    """CUDA graphs of a shape-static launch sequence `fn(*args)` of a model (the fused training step, the no-grad forward), one per
    input signature, the least recently used dropped beyond `capacity` (every captured graph owns a private memory pool).

    The first call of a signature runs eagerly (it allocates the workspace, RoPE tables and split-K scratch and sets kernel
    attributes), the second captures `fn` on static copies of the inputs (kernel arguments, TMA descriptors included, are baked in)
    and every later call copies its inputs into those buffers and replays.  Sharded bf16 frozen weights and shards gathered by NCCL
    (side-stream all-gathers) and non-CUDA models run eagerly; so does a cache whose capture failed once (with a warning: never
    silently wrong).  Sharded NF4 / FP8 codes gathered by peer copies are captured (the copies become memcpy nodes)."""

    def __init__(self, capacity: int, what: str):
        self.capacity, self.what = capacity, what
        self.entries = {}  # key -> "warm" (seen once) | captured graph; most recently used last
        self.failed = False

    def captured(self) -> int:
        return sum(isinstance(e, dict) for e in self.entries.values())

    def clear(self):
        self.entries.clear()

    def run(self, model, fn, args, tag=None, enabled=True):
        """fn(*args) through the graph of key (input signature, tag)."""
        sharded = model._sharded is not None and not getattr(model._sharded, "capturable", False)
        if not enabled or self.failed or sharded or model.dev.type != "cuda" or not torch.cuda.is_available():
            return fn(*args)
        key = (_graph_sig(args), tag, torch.are_deterministic_algorithms_enabled())  # never replay across the two kernel choices
        ent = self.entries.pop(key, None)
        if ent is None:
            while len(self.entries) >= self.capacity:
                self.entries.pop(next(iter(self.entries)))
            self.entries[key] = "warm"
            return fn(*args)
        self.entries[key] = ent
        if ent != "warm" and ent["ws"] is not model._ws and not model._activate_ws(ent["ws"], ent["ws_key"]):
            ent = "warm"  # the model dropped the workspace this graph was recorded on (another shape ran in between): record again
        if ent != "warm" and ent["grad_ptr"] != _grad_ptr(model):
            ent = "warm"  # the gradient accumulator moved (into peer memory, sharding.GradExchange): record again
        if ent == "warm":
            static = _graph_clone(args)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            n0 = lib.LAUNCHES
            try:
                with torch.cuda.graph(g):
                    out = fn(*static)
            except Exception as e:
                warnings.warn(f"qflux_b200: CUDA-graph capture of {self.what} failed ({type(e).__name__}: {e}); running eagerly")
                torch.cuda.synchronize()
                self.failed = True
                lib.LAUNCHES = n0
                return fn(*args)
            # `keep`: per-shape tables the captured kernels point at (RoPE, key lengths, ragged row bands) live in bounded caches of the
            # model — the graph must keep them alive after they are evicted there
            ent = dict(graph=g, static=static, out=out, launches=lib.LAUNCHES - n0, ws=model._ws, ws_key=model._ws_key,
                       grad_ptr=_grad_ptr(model), keep=tuple(model._ws.get(k) for k in ("rope", "kv_len", "txt_len", "bands")))
            lib.LAUNCHES = n0  # capture launches nothing
            self.entries[key] = ent
        _graph_copy(ent["static"], args)
        ent["graph"].replay()
        lib.LAUNCHES += ent["launches"]
        model._fwd_gen += 1  # a replay is a forward that bypasses _forward_impl: autograd nodes of older forwards must refuse to run
        return ent["out"]


def _grad_ptr(model):
    g = getattr(model, "G32", None)  # None before an adapter exists
    return 0 if g is None else g.data_ptr()


def _graph_sig(a):
    if torch.is_tensor(a):
        return ("t", tuple(a.shape), str(a.dtype))
    if isinstance(a, (tuple, list)):
        return tuple(_graph_sig(x) for x in a)
    return repr(a)


def _graph_clone(args):
    return tuple(a.clone() if torch.is_tensor(a) else (_graph_clone(a) if isinstance(a, tuple) else a) for a in args)


def _graph_copy(static, args):
    for s_, a in zip(static, args):
        if torch.is_tensor(s_):
            if s_.data_ptr() != a.data_ptr():
                s_.copy_(a, non_blocking=True)
        elif isinstance(s_, tuple):
            _graph_copy(s_, a)


class ModelFn(torch.autograd.Function):
    """Autograd bridge for `dit(...)`: forward = fused kernels (activations kept in the model workspace), backward = fused
    kernels writing LoRA gradients into the flat accumulator; the returned per-parameter grads are views of it."""

    @staticmethod
    def forward(ctx, model, fwd_args, *params):
        ctx.model = model
        out = model._forward_impl(*fwd_args, train=True).clone()
        ctx.gen = model._fwd_gen  # the activations live in the model's single workspace: a later forward invalidates this graph
        return out

    @staticmethod
    def backward(ctx, dpred):
        m = ctx.model
        if ctx.gen != m._fwd_gen:
            raise RuntimeError("qflux_b200: backward() of a forward whose activations were overwritten by a later forward of the same "
                               "model (one workspace per model: call backward before the next forward)")
        m.G32.zero_()
        m._backward_impl(dpred.to(BF).reshape(-1, m.C_out).contiguous())
        views = m.lora_grad_views(m.G32.to(BF))
        return (None, None) + tuple(views[k] for k in m._lora_params)
