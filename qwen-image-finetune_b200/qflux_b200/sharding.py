"""Sharded frozen weights for the fused MMDiT (SURVEY.md §8e, BASELINE config 4: "FSDP bf16, 8 x B200").

Mirrors what the reference's FSDP branch does to the transformer (/root/reference/src/qflux/trainer/base_trainer.py:333-382):
the FROZEN block weights are split 1/world per rank and a block's full weights exist only while that block runs; the LoRA
parameters are excluded from sharding (`ignored_modules`, :340-342) and their gradients are all-reduced exactly as in data
parallel mode.  B200-first layout instead of FSDP's per-module flat parameters:

  * all per-block tensors of one block (q|k|v, out, up, down, modulation linears, biases, q/k norm weights; both streams) are
    packed into ONE contiguous row of a [L, N_blk] matrix, so a block is ONE collective: all_gather_into_tensor of N_blk/world
    elements per rank (Qwen-Image: 680 MB per block) — not one per nn.Module;
  * two gather buffers ping-pong; the gather of block l+1 (l-1 in the backward) is issued on a side stream before block l
    starts, so NVLink traffic overlaps the ~6 ms of tensor-core work of a block;
  * on one node the gather is NOT a collective: the weights are frozen, so every rank exports its shard once through CUDA IPC
    (include/qfx.h qfx_peer_*) and a block is assembled by `world` copy-engine pulls over NVLink (cudaMemcpyAsync from the mapped
    peer pointers, starting at the next rank so the NVSwitch ports are loaded evenly).  No SM is taken from the GEMMs (an NCCL
    all-gather runs kernels that would) and no rank waits
    for another.  `gather="nccl"` (or QFX_SHARD_GATHER=nccl, or ranks on different hosts) keeps the all_gather_into_tensor path;
  * kernels keep reading plain row-major [out, in] views — the views now point into the gather buffer of the block's slot.
"""
from __future__ import annotations

import os

import torch
import torch.distributed as dist

ALIGN = 128  # elements (256 B): every packed tensor starts on a TMA-friendly boundary


class LayerRing:
    """Stands in for a layer-stacked weight tensor `[L, ...]`: indexing with a layer number returns the view inside the gather
    buffer that currently holds that layer (and fails loudly if it does not)."""

    def __init__(self, owner: "ShardedBlocks", offset: int, shape: tuple):
        self.owner, self.offset, self.shape = owner, offset, tuple(shape)
        self.numel = 1
        for d in shape:
            self.numel *= d

    def __getitem__(self, idx):
        rest = ()
        if isinstance(idx, tuple):
            idx, rest = idx[0], idx[1:]
        slot = self.owner.slot_of(int(idx))
        v = self.owner.gbuf[slot, self.offset: self.offset + self.numel].view(self.shape)
        return v[rest] if rest else v


class ShardedBlocks:
    def __init__(self, stacked: dict, n_layers: int, group=None, gather: str = "auto"):
        """stacked: {name: tensor [L, ...]} (full copies; released by the caller afterwards).
        gather: "auto" (peer copies when every rank is a CUDA device of this host, else NCCL), "peer", or "nccl"."""
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.L = n_layers
        any_t = next(iter(stacked.values()))
        self.dev, self.dtype = any_t.device, any_t.dtype
        off, self.rings = 0, {}
        for name, t in stacked.items():
            assert t.shape[0] == n_layers
            self.rings[name] = LayerRing(self, off, t.shape[1:])
            off += -(-self.rings[name].numel // ALIGN) * ALIGN
        q = self.world * ALIGN
        self.n_blk = -(-off // q) * q
        self.n_shard = self.n_blk // self.world
        self.cuda = self.dev.type == "cuda"
        self.gather = self._pick_gather(os.environ.get("QFX_SHARD_GATHER", gather))
        self._peer_buf, self._peer_ptrs = None, None
        if self.gather == "peer":
            from . import lib
            self._peer_buf = lib.PeerBuffer(n_layers * self.n_shard * self.dtype.itemsize, self.dev)
            self.shard = self._peer_buf.tensor(self.dtype, (n_layers, self.n_shard))
            self.shard.zero_()
        else:
            self.shard = torch.zeros(n_layers, self.n_shard, device=self.dev, dtype=self.dtype)
        lo, hi = self.rank * self.n_shard, (self.rank + 1) * self.n_shard
        for name, t in stacked.items():
            r = self.rings[name]
            a, b = max(lo, r.offset), min(hi, r.offset + r.numel)
            if a < b:
                self.shard[:, a - lo: b - lo] = t.reshape(n_layers, -1)[:, a - r.offset: b - r.offset]
        self.gbuf = torch.zeros(2, self.n_blk, device=self.dev, dtype=self.dtype)
        self.in_slot = [None, None]
        if self.gather == "peer":
            self._open_peers()
        if self.cuda:
            self.comm = torch.cuda.Stream(device=self.dev)
            self.ready = [torch.cuda.Event(), torch.cuda.Event()]     # gather into slot finished (comm stream)
            self.released = [torch.cuda.Event(), torch.cuda.Event()]  # last reader of the slot finished (compute stream)
            for e in self.released:
                e.record()
        self.pending = [False, False]

    # ------------------------------------------------------------------------------------------------------------
    def slot_of(self, l: int) -> int:
        s = l & 1
        if self.in_slot[s] != l:
            raise RuntimeError(f"block {l} is not resident (slot {s} holds {self.in_slot[s]}): call acquire({l}) first")
        return s

    def prefetch(self, l: int):
        """Start gathering block l into its slot (no-op if it is there already or l is out of range)."""
        if l < 0 or l >= self.L or self.in_slot[l & 1] == l:
            return
        s = l & 1
        if self.cuda:
            self.comm.wait_event(self.released[s])  # the previous occupant's kernels have finished reading
            with torch.cuda.stream(self.comm):
                self._gather(s, l)
                self.ready[s].record(self.comm)
            self.pending[s] = True
        else:
            self._gather(s, l)
        self.in_slot[s] = l

    def _gather(self, s: int, l: int):
        if self.world == 1:
            self.gbuf[s].copy_(self.shard[l])
        elif self.gather == "peer":
            from . import lib
            nb = self.n_shard * self.dtype.itemsize
            dst = self.gbuf[s].data_ptr()
            for i in range(self.world):  # own shard last; the pulls start at the next rank so no port sees all ranks at once
                r = (self.rank + 1 + i) % self.world
                lib.peer_copy_async(dst + r * nb, self._peer_ptrs[r] + l * nb, nb)
        else:
            dist.all_gather_into_tensor(self.gbuf[s], self.shard[l], group=self.group)

    # ------------------------------------------------------------------------------------------------------------
    def _pick_gather(self, want: str) -> str:
        if want not in ("auto", "peer", "nccl"):
            raise ValueError(f"gather must be auto|peer|nccl, got {want!r}")
        if self.world == 1 or not self.cuda:
            if want == "peer" and self.world > 1:
                raise RuntimeError("gather='peer' needs CUDA devices")
            return "nccl"
        if want == "nccl":
            return "nccl"
        import socket
        hosts = [None] * self.world
        dist.all_gather_object(hosts, socket.gethostname(), group=self.group)
        one_host = len(set(hosts)) == 1
        if want == "peer" and not one_host:
            raise RuntimeError(f"gather='peer' needs all ranks on one host (CUDA IPC); got {sorted(set(hosts))}")
        return "peer" if one_host else "nccl"

    def _open_peers(self):
        """Exchange the IPC handles and map every other rank's shard.  The shards are written before this point and never again
        (frozen weights), so one barrier makes them visible and the data path needs no further cross-rank synchronisation."""
        from . import lib
        torch.cuda.synchronize(self.dev)
        handles = [None] * self.world
        dist.all_gather_object(handles, self._peer_buf.handle, group=self.group)
        self._peer_ptrs = [self._peer_buf.ptr if r == self.rank else lib.peer_open(handles[r], self.dev) for r in range(self.world)]
        dist.barrier(group=self.group)

    def close(self):
        """Unmap the peers' shards and free this rank's (collective: every rank must call it)."""
        if self._peer_ptrs is not None:
            from . import lib
            torch.cuda.synchronize(self.dev)
            for r, p in enumerate(self._peer_ptrs):
                if r != self.rank:
                    lib.peer_close(p)
            self._peer_ptrs = None
            dist.barrier(group=self.group)
            self.shard = None
            self._peer_buf.free()

    def acquire(self, l: int):
        """Make block l's weights valid for kernels on the current stream."""
        self.prefetch(l)
        s = l & 1
        if self.cuda and self.pending[s]:
            torch.cuda.current_stream().wait_event(self.ready[s])
            self.pending[s] = False

    def release(self, l: int):
        """The kernels of block l have been enqueued on the current stream; its slot may be refilled once they finish."""
        if self.cuda:
            self.released[l & 1].record(torch.cuda.current_stream())
