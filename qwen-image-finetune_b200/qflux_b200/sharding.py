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

The same two-slot ring (`BlockRing`) has two more fill sources: `Nf4Blocks` dequantizes a block's NF4-resident matrices
(4-bit base checkpoints, nf4.py) into its slot with one kernel launch, and `Fp8Blocks` expands its FP8-resident matrices
(float8-e4m3fn base checkpoints, fp8.py) the same way.
"""
from __future__ import annotations

import os

import torch
import torch.distributed as dist

ALIGN = 128  # elements (256 B): every packed tensor starts on a TMA-friendly boundary


class LayerRing:
    """Stands in for a layer-stacked weight tensor `[L, ...]`: indexing with a layer number returns the view inside the ring
    buffer slot that currently holds that layer (and fails loudly if it does not)."""

    def __init__(self, owner: "BlockRing", offset: int, shape: tuple):
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


class BlockRing:
    """Two-slot ring of one block kind's weights: block l is filled into slot l & 1 on a side stream (`prefetch`), kernels on
    the compute stream wait for it (`acquire`), and the slot is refilled only after its last reader has finished (`release`).
    Subclasses provide the fill source (`_fill(slot, l)`): an all-gather of the ranks' shards, the NF4 dequantization or the FP8 expansion."""

    def _layout(self, shapes: dict, n_layers: int, dev, dtype) -> int:
        """One LayerRing view per tensor, each starting on an ALIGN boundary of the slot.  Returns the elements a slot needs."""
        self.L, self.dev, self.dtype, self.cuda = n_layers, dev, dtype, dev.type == "cuda"
        off, self.rings = 0, {}
        for name, shape in shapes.items():
            self.rings[name] = LayerRing(self, off, shape)
            off += -(-self.rings[name].numel // ALIGN) * ALIGN
        return off

    def _alloc_slots(self, n_blk: int):
        self.gbuf = torch.zeros(2, n_blk, device=self.dev, dtype=self.dtype)
        self.in_slot = [None, None]
        if self.cuda:
            self.comm = torch.cuda.Stream(device=self.dev)
            self.ready = [torch.cuda.Event(), torch.cuda.Event()]     # fill of the slot finished (comm stream)
            self.released = [torch.cuda.Event(), torch.cuda.Event()]  # last reader of the slot finished (compute stream)
            for e in self.released:
                e.record()
        self.pending = [False, False]

    def _fill(self, s: int, l: int):
        raise NotImplementedError

    # ------------------------------------------------------------------------------------------------------------
    def slot_of(self, l: int) -> int:
        s = l & 1
        if self.in_slot[s] != l:
            raise RuntimeError(f"block {l} is not resident (slot {s} holds {self.in_slot[s]}): call acquire({l}) first")
        return s

    def prefetch(self, l: int):
        """Start filling block l into its slot (no-op if it is there already or l is out of range)."""
        if l < 0 or l >= self.L or self.in_slot[l & 1] == l:
            return
        s = l & 1
        if self.cuda:
            self.comm.wait_event(self.released[s])  # the previous occupant's kernels have finished reading
            with torch.cuda.stream(self.comm):
                self._fill(s, l)
                self.ready[s].record(self.comm)
            self.pending[s] = True
        else:
            self._fill(s, l)
        self.in_slot[s] = l

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

    def join(self):
        """The current stream waits for everything issued on the side stream (the end of a captured region must join every stream
        that forked from it)."""
        if self.cuda:
            torch.cuda.current_stream().wait_stream(self.comm)

    def reset(self):
        """Forget what the slots hold; the next fills wait for everything enqueued so far on the current stream.  A forward that
        starts here fills the same blocks whether it runs eagerly or is captured into a CUDA graph and replayed, and under capture
        the side stream forks from the capturing stream through events recorded inside the capture (and joins it again in
        `acquire`)."""
        self.in_slot, self.pending = [None, None], [False, False]
        if self.cuda:
            for e in self.released:
                e.record(torch.cuda.current_stream())


class ShardedBlocks(BlockRing):
    def __init__(self, stacked: dict, n_layers: int, group=None, gather: str = "auto"):
        """stacked: {name: tensor [L, ...]} (full copies; released by the caller afterwards).
        gather: "auto" (peer copies when every rank is a CUDA device of this host, else NCCL), "peer", or "nccl"."""
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        any_t = next(iter(stacked.values()))
        for t in stacked.values():
            assert t.shape[0] == n_layers
        off = self._layout({name: t.shape[1:] for name, t in stacked.items()}, n_layers, any_t.device, any_t.dtype)
        q = self.world * ALIGN
        self.n_blk = -(-off // q) * q
        self.n_shard = self.n_blk // self.world
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
        self._alloc_slots(self.n_blk)
        if self.gather == "peer":
            self._open_peers()

    def _fill(self, s: int, l: int):
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


class GradExchange:
    """Bit-reproducible data-parallel sum of the flat fp32 LoRA gradient `G32`: what `train_step._sync_and_step` runs in place of
    `all_reduce(G32)` under torch.use_deterministic_algorithms(True) when every rank is a CUDA device of this host.  Element i of the
    result is ((((+0) + g_0[i]) + g_1[i]) + ...) + g_{W-1}[i] in rank order (qfx_dp_reduce_det), the same bits on every rank:

      1. reduce-scatter: rank q sums slice q of every rank's G32, read in place through CUDA IPC, into slice q of its own G32;
      2. all-gather: rank q pulls every other rank's reduced slice with the copy engines, starting at the next rank.

    Each rank moves 2 (W - 1) / W of the buffer, as a ring all-reduce does.  Nothing is allocated per step: the first exchange moves
    G32 itself into an IPC-exportable allocation.  Three points order the ranks' streams: before the reduce (every G32 is final),
    before the gather (every slice is reduced) and after it (every peer has pulled this rank's slices, so the next backward may write
    G32 again).  At each, every rank records an interprocess CUDA event, a barrier on a gloo group guarantees that every rank has issued
    its record, and the stream waits for the peers' events: the host never waits for the device and no kernel waits for another process.

    CPU models (the emulated kernels of the gloo tests) run the same two phases with dist.all_gather in place of the peer reads."""

    @staticmethod
    def for_model(model):
        """The model's exchange, set up by its first call (collective); None when the ranks are not all on this host with the same
        kind of device."""
        ex = getattr(model, "_grad_exchange", None)
        if ex is None:
            import socket
            where = [None] * dist.get_world_size()
            dist.all_gather_object(where, (socket.gethostname(), model.dev.type))
            ex = model._grad_exchange = GradExchange(model) if len(set(where)) == 1 else False
        return ex or None

    def __init__(self, model):
        self.model, self.dev, self.cuda = model, model.dev, model.dev.type == "cuda"
        self.world, self.rank = dist.get_world_size(), dist.get_rank()
        self.host = dist.group.WORLD if dist.get_backend() == "gloo" else dist.new_group(backend="gloo")
        n = model.G32.numel()
        c = -(-n // (self.world * ALIGN)) * ALIGN  # slice q = [q c, (q + 1) c), 512-byte aligned (the last may be short or empty)
        self.bounds = [(min(n, q * c), min(n, (q + 1) * c)) for q in range(self.world)]
        self._buf = None
        if self.cuda:
            self._open()

    def _open(self):
        from . import lib
        with torch.cuda.device(self.dev):
            self._buf = lib.PeerBuffer(self.model.G32.numel() * 4, self.dev)
            g32 = self._buf.tensor(torch.float32, (self.model.G32.numel(),))
            g32.copy_(self.model.G32)
            self.model.G32 = g32
            torch.cuda.empty_cache()  # the old accumulator's memory goes back to the device
            self._events = [torch.cuda.Event(interprocess=True) for _ in range(3)]  # G32 final, slice reduced, peers' slices pulled
            for e in self._events:
                e.record()
            mine = (self._buf.handle, [e.ipc_handle() for e in self._events])
            peers = [None] * self.world
            dist.all_gather_object(peers, mine, group=self.host)
            self._ptrs = [self._buf.ptr if r == self.rank else lib.peer_open(peers[r][0], self.dev) for r in range(self.world)]
            self._peer_events = [[torch.cuda.Event.from_ipc_handle(self.dev, h) for h in peers[r][1]]
                                 for r in range(self.world) if r != self.rank]
        dist.barrier(group=self.host)

    def _point(self, k: int):
        s = torch.cuda.current_stream(self.dev)
        self._events[k].record(s)
        dist.barrier(group=self.host)  # every rank has issued its record k: the waits below see this step's
        for evs in self._peer_events:
            s.wait_event(evs[k])

    def all_reduce(self):
        """G32 <- the rank-ordered sum of every rank's G32 (collective; asynchronous on the current stream)."""
        from . import lib
        g32 = self.model.G32
        if not self.cuda:
            bufs = [torch.empty_like(g32) for _ in range(self.world)]
            dist.all_gather(bufs, g32, group=self.host)
            lo, hi = self.bounds[self.rank]
            if hi > lo:
                lib.dp_reduce_det([b[lo:hi] for b in bufs], g32[lo:hi])
            dist.all_gather(bufs, g32, group=self.host)
            for r, (lo, hi) in enumerate(self.bounds):
                if r != self.rank:
                    g32[lo:hi] = bufs[r][lo:hi]
            return
        if g32.data_ptr() != self._buf.ptr:
            raise RuntimeError("GradExchange: the model's G32 was replaced after the exchange was set up (add_adapter during "
                               "data-parallel training); call model.close() on every rank first")
        with torch.cuda.device(self.dev):
            self._point(0)
            lo, hi = self.bounds[self.rank]
            if hi > lo:
                lib.dp_reduce_det([p + lo * 4 for p in self._ptrs], g32[lo:hi])
            self._point(1)
            for i in range(1, self.world):
                r = (self.rank + i) % self.world
                lo, hi = self.bounds[r]
                if hi > lo:
                    lib.peer_copy_async(self._buf.ptr + lo * 4, self._ptrs[r] + lo * 4, (hi - lo) * 4)
            self._point(2)

    def close(self):
        """Unmap the peers' gradients and move G32 back into an ordinary allocation (collective: every rank must call it)."""
        if self._buf is None:
            return
        from . import lib
        with torch.cuda.device(self.dev):
            g32 = self.model.G32.clone()
            torch.cuda.synchronize(self.dev)  # the last exchange's reads of the peers' memory have finished
            for r, p in enumerate(self._ptrs):
                if r != self.rank:
                    lib.peer_close(p)
            dist.barrier(group=self.host)
            self.model.G32 = g32
            self._buf.free()
            self._buf = None


class Nf4Blocks(BlockRing):
    """NF4-resident frozen weights: every NF4 matrix of a block kind lives as layer-stacked codes + fp32 absmax (nf4.py); a block's
    bf16 matrices are produced in its ring slot by ONE qfx_nf4_dequant launch right before it runs.  Kernels read the same
    row-major [out, in] bf16 views as for resident or sharded weights."""

    def __init__(self, stacks: dict, n_layers: int, blocksize: int):
        """stacks: {name: (codes uint8 [L, ..., in/2], absmax fp32 [L, n/blocksize], bf16 shape of one layer)}."""
        codes0 = next(iter(stacks.values()))[0]
        off = self._layout({k: shape for k, (_, _, shape) in stacks.items()}, n_layers, codes0.device, torch.bfloat16)
        self.stacks, self.blocksize = stacks, blocksize
        self._alloc_slots(off)

    def _fill(self, s: int, l: int):
        from . import lib
        lib.nf4_dequant([(c[l].reshape(-1), a[l].reshape(-1), self.gbuf[s, self.rings[k].offset: self.rings[k].offset + self.rings[k].numel],
                          self.blocksize) for k, (c, a, _) in self.stacks.items()])


class Fp8Blocks(BlockRing):
    """FP8-resident frozen weights: every FP8 matrix of a block kind lives as layer-stacked float8-e4m3fn codes (fp8.py), one byte
    per element in the bf16 layout; a block's bf16 matrices are produced in its ring slot by ONE qfx_fp8_expand launch right before
    it runs (exact: every finite e4m3fn value is a bf16 value)."""

    def __init__(self, stacks: dict, n_layers: int):
        """stacks: {name: codes float8_e4m3fn [L, ...] (the bf16 shape of the stack)}."""
        codes0 = next(iter(stacks.values()))
        off = self._layout({k: tuple(c.shape[1:]) for k, c in stacks.items()}, n_layers, codes0.device, torch.bfloat16)
        self.stacks = stacks
        self._alloc_slots(off)

    def _fill(self, s: int, l: int):
        from . import lib
        lib.fp8_expand([(c[l].reshape(-1), self.gbuf[s, self.rings[k].offset: self.rings[k].offset + self.rings[k].numel])
                        for k, c in self.stacks.items()])
