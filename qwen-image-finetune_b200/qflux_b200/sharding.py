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

The same two-slot ring (`BlockRing`) has more fill sources: `Nf4Blocks` dequantizes a block's NF4-resident matrices
(4-bit base checkpoints, nf4.py) into its slot with one kernel launch, and `Fp8Blocks` expands its FP8-resident matrices
(float8-e4m3fn base checkpoints, fp8.py) the same way.  `ShardedNf4Blocks` / `ShardedFp8Blocks` shard those codes across the
ranks: a block's code bytes are gathered as above (`ShardGather`, shared with `ShardedBlocks`) into a staging slot, then expanded
from there by the same launch.
"""
from __future__ import annotations

import bisect
import contextlib
import os

import torch
import torch.distributed as dist

ALIGN = 128  # elements (256 B): every packed tensor starts on a TMA-friendly boundary
ALIGN_BYTES = 2 * ALIGN  # the same boundary for rows of any element type (sharded rows are padded to it per rank)


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


class ShardGather:
    """The gather half of a sharded ring: this rank keeps columns [rank n_shard, (rank + 1) n_shard) of a layer-stacked [L, n_blk]
    matrix whose rows are the packed blocks, and `_pull(dst, l)` assembles row l into dst on the current stream.  On one host every
    rank exports its shard once through CUDA IPC and a row is `world` copy-engine pulls from the mapped peer pointers, starting at the
    next rank; otherwise (or with gather="nccl") it is one all_gather_into_tensor.  Used by ShardedBlocks (bf16 rows) and by
    ShardedNf4Blocks / ShardedFp8Blocks (rows of NF4 / FP8 code bytes)."""

    def _init_shards(self, parts, n_row: int, n_layers: int, dtype, group, gather: str):
        """parts: [(offset in the row, tensor [L, n] of `dtype`)], the row segments (full copies; released by the caller afterwards).
        The row is padded to whole ALIGN_BYTES per rank.  gather: "auto" (peer copies when every rank is a CUDA device of this host,
        else NCCL), "peer", or "nccl".  Collective."""
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        q = self.world * (ALIGN_BYTES // dtype.itemsize)
        self.n_blk = -(-n_row // q) * q
        self.n_shard = self.n_blk // self.world
        self.gather = self._pick_gather(os.environ.get("QFX_SHARD_GATHER", gather))
        self._peer_buf, self._peer_ptrs = None, None
        if self.gather == "peer":
            from . import lib
            self._peer_buf = lib.PeerBuffer(n_layers * self.n_shard * dtype.itemsize, self.dev)
            self.shard = self._peer_buf.tensor(dtype, (n_layers, self.n_shard))
            self.shard.zero_()
        else:
            self.shard = torch.zeros(n_layers, self.n_shard, device=self.dev, dtype=dtype)
        lo, hi = self.rank * self.n_shard, (self.rank + 1) * self.n_shard
        for off, t in parts:
            a, b = max(lo, off), min(hi, off + t.shape[1])
            if a < b:
                self.shard[:, a - lo: b - lo] = t[:, a - off: b - off]
        if self.gather == "peer":
            self._open_peers()

    @property
    def capturable(self) -> bool:
        """Whether a forward through this ring may be captured into a CUDA graph (GraphCache)."""
        return False

    def _pull(self, dst, l: int):
        """dst (the [n_blk] row buffer) <- row l, assembled from every rank's shard on the current stream."""
        if self.world == 1:
            dst.copy_(self.shard[l])
        elif self.gather == "peer":
            from . import lib
            nb = self.n_shard * self.shard.element_size()
            for i in range(self.world):  # own shard last; the pulls start at the next rank so no port sees all ranks at once
                r = (self.rank + 1 + i) % self.world
                lib.peer_copy_async(dst.data_ptr() + r * nb, self._peer_ptrs[r] + l * nb, nb)
        else:
            dist.all_gather_into_tensor(dst, self.shard[l], group=self.group)

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


class ShardedBlocks(ShardGather, BlockRing):
    def __init__(self, stacked: dict, n_layers: int, group=None, gather: str = "auto"):
        """stacked: {name: tensor [L, ...]} (full copies; released by the caller afterwards).
        gather: "auto" (peer copies when every rank is a CUDA device of this host, else NCCL), "peer", or "nccl"."""
        any_t = next(iter(stacked.values()))
        for t in stacked.values():
            assert t.shape[0] == n_layers
        off = self._layout({name: t.shape[1:] for name, t in stacked.items()}, n_layers, any_t.device, any_t.dtype)
        self._init_shards([(self.rings[name].offset, t.reshape(n_layers, -1)) for name, t in stacked.items()], off, n_layers,
                          self.dtype, group, gather)
        self._alloc_slots(self.n_blk)

    def _fill(self, s: int, l: int):
        self._pull(self.gbuf[s], l)


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

    def _reduce_slice(self, bounds):
        """Phase 1 with slice q = bounds[q]: this rank's slice of G32 <- the rank-ordered sum of every rank's slice.  Returns the
        gathered copies of every rank's G32 on CPU models (phase 2 reuses them)."""
        from . import lib
        g32 = self.model.G32
        lo, hi = bounds[self.rank]
        if not self.cuda:
            bufs = [torch.empty_like(g32) for _ in range(self.world)]
            dist.all_gather(bufs, g32, group=self.host)
            if hi > lo:
                lib.dp_reduce_det([b[lo:hi] for b in bufs], g32[lo:hi])
            return bufs
        if g32.data_ptr() != self._buf.ptr:
            raise RuntimeError("GradExchange: the model's G32 was replaced after the exchange was set up (add_adapter during "
                               "data-parallel training); call model.close() on every rank first")
        self._point(0)
        if hi > lo:
            lib.dp_reduce_det([p + lo * 4 for p in self._ptrs], g32[lo:hi])
        self._point(1)
        return None

    def reduce_scatter(self, bounds):
        """Slice bounds[rank] of G32 <- the rank-ordered sum of every rank's G32 there; the rest of G32 is left as it is (collective;
        asynchronous on the current stream).  The sharded optimizer's exchange: phase 1 without the all-gather.  The point after the
        reduce also orders the next write of G32 after every peer's reads of it."""
        with torch.cuda.device(self.dev) if self.cuda else contextlib.nullcontext():
            self._reduce_slice(bounds)

    def all_reduce(self):
        """G32 <- the rank-ordered sum of every rank's G32 (collective; asynchronous on the current stream)."""
        from . import lib
        g32 = self.model.G32
        if not self.cuda:
            bufs = self._reduce_slice(self.bounds)
            dist.all_gather(bufs, g32, group=self.host)
            for r, (lo, hi) in enumerate(self.bounds):
                if r != self.rank:
                    g32[lo:hi] = bufs[r][lo:hi]
            return
        with torch.cuda.device(self.dev):
            self._reduce_slice(self.bounds)
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


class CodeBlocks(BlockRing):
    """A ring filled by expanding a block's resident codes: `codes` holds {kind: (layer-stacked code tensors [L, ...] of one matrix)},
    and `_expand(s, src)` fills slot s from {kind: (the flat code tensors of one layer)} in ONE launch (the segment table).  The
    sources are the resident stacks here, a staging slot of gathered shards in ShardedCodes."""

    def _layer_codes(self, l: int) -> dict:
        return {k: tuple(t[l].reshape(-1) for t in ts) for k, ts in self.codes.items()}

    def _out(self, s: int, k: str):
        r = self.rings[k]
        return self.gbuf[s, r.offset: r.offset + r.numel]

    def _expand(self, s: int, src: dict):
        raise NotImplementedError

    def _fill(self, s: int, l: int):
        self._expand(s, self._layer_codes(l))


class Nf4Blocks(CodeBlocks):
    """NF4-resident frozen weights: every NF4 matrix of a block kind lives as layer-stacked codes + fp32 absmax (nf4.py); a block's
    bf16 matrices are produced in its ring slot by ONE qfx_nf4_dequant launch right before it runs.  Kernels read the same
    row-major [out, in] bf16 views as for resident or sharded weights."""

    def __init__(self, stacks: dict, n_layers: int, blocksize: int):
        """stacks: {name: (codes uint8 [L, ..., in/2], absmax fp32 [L, n/blocksize], bf16 shape of one layer)}."""
        codes0 = next(iter(stacks.values()))[0]
        off = self._layout({k: shape for k, (_, _, shape) in stacks.items()}, n_layers, codes0.device, torch.bfloat16)
        self.codes, self.blocksize = {k: (c, a) for k, (c, a, _) in stacks.items()}, blocksize
        self._alloc_slots(off)

    def _expand(self, s: int, src: dict):
        from . import lib
        lib.nf4_dequant([(c, a, self._out(s, k), self.blocksize) for k, (c, a) in src.items()])


class Fp8Blocks(CodeBlocks):
    """FP8-resident frozen weights: every FP8 matrix of a block kind lives as layer-stacked float8-e4m3fn codes (fp8.py), one byte
    per element in the bf16 layout; a block's bf16 matrices are produced in its ring slot by ONE qfx_fp8_expand launch right before
    it runs (exact: every finite e4m3fn value is a bf16 value)."""

    def __init__(self, stacks: dict, n_layers: int):
        """stacks: {name: codes float8_e4m3fn [L, ...] (the bf16 shape of the stack)}."""
        codes0 = next(iter(stacks.values()))
        off = self._layout({k: tuple(c.shape[1:]) for k, c in stacks.items()}, n_layers, codes0.device, torch.bfloat16)
        self.codes = {k: (c,) for k, c in stacks.items()}
        self._alloc_slots(off)

    def _expand(self, s: int, src: dict):
        from . import lib
        lib.fp8_expand([(c, self._out(s, k)) for k, (c,) in src.items()])


class ShardedCodes(ShardGather):
    """Sharded NF4 / FP8 frozen weights: the resident codes of one block (every NF4 matrix's uint8 codes and fp32 absmax, or every
    FP8 matrix's e4m3fn bytes) are packed into ONE byte row, each tensor on an ALIGN_BYTES boundary, and this rank keeps 1/world of
    every layer's row (ShardGather).  A block is filled in two stages on the ring's side stream: the W shards of its row are gathered
    into a per-slot staging buffer, then ONE expansion launch (the subclass's `_expand`, the same segment table as for resident codes)
    runs from the staging slot into the bf16 slot.  Both stages are ordered by the ring's prefetch / acquire / release events, so the
    block kernels read the same bf16 views as for resident codes; the peer pulls are copies, so a forward through the ring can be
    captured into a CUDA graph (memcpy nodes), the NCCL all-gather cannot."""

    def _shard_codes(self, group, gather):
        """Replace `codes` by this rank's shard of the packed rows and allocate the two staging slots (collective)."""
        row, parts, off = {}, [], 0
        for k, ts in self.codes.items():
            row[k] = []
            for t in ts:
                flat = t.reshape(self.L, -1)
                row[k].append((off, flat.shape[1], t.dtype))
                parts.append((off, flat.view(torch.uint8)))
                off += -(-flat.shape[1] * t.element_size() // ALIGN_BYTES) * ALIGN_BYTES
        self._init_shards(parts, off, self.L, torch.uint8, group, gather)
        self.codes = None  # the full stacks are the caller's to free
        self.stage = torch.zeros(2, self.n_blk, device=self.dev, dtype=torch.uint8)
        # the segment tables' sources: every code tensor of a block as a view into each staging slot
        self._staged = [{k: tuple(self.stage[s, o: o + n * dt.itemsize].view(dt) for o, n, dt in segs) for k, segs in row.items()}
                        for s in range(2)]

    @property
    def capturable(self) -> bool:
        return self.gather == "peer"

    def _fill(self, s: int, l: int):
        self._pull(self.stage[s], l)
        self._expand(s, self._staged[s])


class ShardedNf4Blocks(ShardedCodes, Nf4Blocks):
    def __init__(self, stacks: dict, n_layers: int, blocksize: int, group=None, gather: str = "auto"):
        """stacks: as for Nf4Blocks (full copies; released by the caller afterwards); group / gather: as for ShardedBlocks."""
        Nf4Blocks.__init__(self, stacks, n_layers, blocksize)
        self._shard_codes(group, gather)


class ShardedFp8Blocks(ShardedCodes, Fp8Blocks):
    def __init__(self, stacks: dict, n_layers: int, group=None, gather: str = "auto"):
        """stacks: as for Fp8Blocks (full copies; released by the caller afterwards); group / gather: as for ShardedBlocks."""
        Fp8Blocks.__init__(self, stacks, n_layers)
        self._shard_codes(group, gather)


class SlicePlan:
    """Which part of the flat LoRA gradient each data-parallel rank's sharded optimizer owns (optim.py shard_state=True).

    The members (the optimizer's (LoRA tensor, gradient offset) pairs) are taken in gradient-offset order, `members`, and tiled into
    chunks of <= lib.ADAMW_CHUNK consecutive elements of one tensor, `chunks`, as lib.adamw_tables tiles them; a sharded optimizer
    builds its tables from `members`.  The chunk list is split into `world` contiguous ranges balanced by element count: cut q sits at
    the chunk boundary nearest to q / world of the elements, so every slice is within one chunk of the mean.  Cuts fall on chunk
    boundaries only, so an 8-bit Adam block (256 elements, which divides the chunk) is never cut and every per-chunk Prodigy partial
    belongs to one rank.  Slice q's gradient range `bounds[q]` runs from its first chunk's offset to the next slice's (0 and
    G32.numel() at the ends): the slices partition G32, which keeps its layout.  `order[j]` is the index in the caller's member list
    of `members[j]`, and `table_chunk[c]` the index of chunk c in the chunk list of the caller's order (the replicated optimizer's
    tables).  The exchange, the optimizer's state, its state_dict and the tests all read their slice bounds from here."""

    def __init__(self, members, n_grad: int, world: int):
        from . import lib
        members = list(members)
        self.world, self.n_grad = int(world), int(n_grad)
        self.order = sorted(range(len(members)), key=lambda i: members[i][1])
        self.members = [members[i] for i in self.order]
        first, c = [], 0  # first chunk of each member in the caller's order
        for p, _ in members:
            first.append(c)
            c += -(-p.numel() // lib.ADAMW_CHUNK)
        chunks, table_chunk, end = [], [], 0  # (member, first element, gradient offset, elements)
        for j, (p, off) in enumerate(self.members):
            n = p.numel()
            if off < end or off + n > n_grad:
                raise ValueError("SlicePlan: members must sit in disjoint ranges of the flat gradient")
            chunks += [(j, e, off + e, min(lib.ADAMW_CHUNK, n - e)) for e in range(0, n, lib.ADAMW_CHUNK)]
            table_chunk += [first[self.order[j]] + k for k in range(-(-n // lib.ADAMW_CHUNK))]
            end = off + n
        self.chunks, self.table_chunk = chunks, table_chunk
        prefix = [0]
        for c in chunks:
            prefix.append(prefix[-1] + c[3])
        total, cuts = prefix[-1], [0]
        for q in range(1, world):
            target = total * q / world
            k = bisect.bisect_left(prefix, target, lo=cuts[-1])
            if k > cuts[-1] and (k == len(prefix) or target - prefix[k - 1] <= prefix[k] - target):
                k -= 1
            cuts.append(min(k, len(chunks)))
        cuts.append(len(chunks))
        self.chunk_ranges = [(cuts[q], cuts[q + 1]) for q in range(world)]
        start = [c[2] for c in chunks] + [self.n_grad]
        start[0] = 0
        self.bounds = [(start[c0], start[c1]) for c0, c1 in self.chunk_ranges]
        self._starts = [c[2] for c in chunks]
        self.elements = [prefix[c1] - prefix[c0] for c0, c1 in self.chunk_ranges]

    def pieces(self, q):
        """(index into `members`, first element, end element) of every tensor part in slice q, in gradient order."""
        out = []
        for i, e, _, n in self.chunks[slice(*self.chunk_ranges[q])]:
            if out and out[-1][0] == i and out[-1][2] == e:
                out[-1] = (i, out[-1][1], e + n)
            else:
                out.append((i, e, e + n))
        return out

    def chunks_in(self, q, g_lo, g_hi):
        """The chunk range of slice q whose chunks meet the gradient range [g_lo, g_hi)."""
        c0, c1 = self.chunk_ranges[q]
        a = max(c0, bisect.bisect_right(self._starts, g_lo, c0, c1) - 1)
        b = bisect.bisect_left(self._starts, g_hi, a, c1)
        return (a, max(a, b))


class ShardExchange:
    """The collectives of a sharded fused optimizer (optim.py shard_state=True), in step order:

      * reduce_scatter(): slice q of G32 on rank q <- the sum over ranks.  Under torch.use_deterministic_algorithms(True) with every
        rank on this host, GradExchange's phase 1 (rank-ordered, through peer memory) on the plan's bounds.  Otherwise, with NCCL,
        reduce_scatter_tensor in pieces staged through a fixed buffer (slices padded to the piece length); with gloo, which has no
        reduce-scatter, an all_gather and the rank-ordered sum (qfx_dp_reduce_det), as GradExchange does on CPU models.
      * gather_sum(mine, out): the ranks' fp32 partials (one each) all-gathered and added in rank order into out, on the device.
      * gather_rows(x, rows): x holds this rank's rows [c0, c1) (plan chunk ranges) of a [n_chunks, k] table; the other ranks' rows
        are all-gathered into it.
      * gather_weights(): every rank's updated slice of LoRA weights packed (qfx_lora_pack), all-gathered and unpacked into the other
        ranks' parameter views (qfx_lora_unpack), in pieces of at most STAGING_BYTES.
    Nothing here waits for the device; all of it is on the current stream."""

    STAGING_BYTES = 64 << 20

    def __init__(self, model, plan: SlicePlan, tables):
        self.model, self.plan, self.tables = model, plan, tables
        self.world, self.rank = dist.get_world_size(), dist.get_rank()
        self.nccl = dist.get_backend() == "nccl"
        self.dev = model.dev
        self._stage = None  # STAGING_BYTES, made at the first exchange that needs it

    def _staging(self):
        if self._stage is None:
            self._stage = torch.empty(self.STAGING_BYTES, device=self.dev, dtype=torch.uint8)
        return self._stage

    def reduce_scatter(self):
        from . import lib
        g32, (lo, hi) = self.model.G32, self.plan.bounds[self.rank]
        if torch.are_deterministic_algorithms_enabled():
            ex = GradExchange.for_model(self.model)
            if ex is not None:
                ex.reduce_scatter(self.plan.bounds)
                return
        if not self.nccl:
            bufs = [torch.empty_like(g32) for _ in range(self.world)]
            dist.all_gather(bufs, g32)
            if hi > lo:
                lib.dp_reduce_det([b[lo:hi] for b in bufs], g32[lo:hi])
            return
        P = self.STAGING_BYTES // 4 // (self.world + 1)  # fp32 elements per rank and piece: [world, L] sent, [L] received, L <= P
        stage = self._staging().view(torch.float32)
        longest = max(b - a for a, b in self.plan.bounds)
        for k0 in range(0, longest, P):
            L = min(P, longest - k0)
            send, recv = stage[: self.world * L].view(self.world, L), stage[self.world * P: self.world * P + L]
            for r, (a, b) in enumerate(self.plan.bounds):
                n = max(0, min(L, b - a - k0))
                send[r, :n] = g32[a + k0: a + k0 + n]
                send[r, n:] = 0
            dist.reduce_scatter_tensor(recv, send.view(-1))
            n = max(0, min(L, hi - lo - k0))
            g32[lo + k0: lo + k0 + n] = recv[:n]

    def gather_sum(self, mine, out):
        from . import lib
        parts = torch.empty(self.world, device=mine.device, dtype=torch.float32)
        dist.all_gather_into_tensor(parts, mine.reshape(1))
        lib.dp_reduce_det([parts[r: r + 1] for r in range(self.world)], out.reshape(1))

    def gather_rows(self, x):
        """x: [n_chunks, k] (any dtype) whose rows of this rank's chunk range are current; afterwards every row is."""
        rows = [c1 - c0 for c0, c1 in self.plan.chunk_ranges]
        most = max(rows)
        if most == 0:
            return
        c0, c1 = self.plan.chunk_ranges[self.rank]
        mine = torch.zeros(most, *x.shape[1:], device=x.device, dtype=x.dtype)
        mine[: c1 - c0] = x[c0:c1]
        every = torch.empty(self.world * most, *x.shape[1:], device=x.device, dtype=x.dtype)
        dist.all_gather_into_tensor(every, mine)
        for r, (a, b) in enumerate(self.plan.chunk_ranges):
            if r != self.rank and b > a:
                x[a:b] = every[r * most: r * most + b - a]

    def gather_weights(self):
        from . import lib
        P = self.STAGING_BYTES // 2 // (self.world + 1)  # bf16 elements per rank and piece: [P] packed, [world, P] gathered
        stage = self._staging().view(torch.bfloat16)
        send, recv = stage[:P], stage[P: (self.world + 1) * P]
        plan, q = self.plan, self.rank
        longest = max(b - a for a, b in plan.bounds)
        for k0 in range(0, longest, P):
            L = min(P, longest - k0)
            lo, hi = plan.bounds[q]
            a, b = lo + k0, min(hi, lo + k0 + L)
            if b > a:
                lib.lora_pack(self.tables, plan.chunks_in(q, a, b), a, b, send[: b - a])
            dist.all_gather_into_tensor(recv[: self.world * L], send[:L])
            for r, (lo, hi) in enumerate(plan.bounds):
                a, b = lo + k0, min(hi, lo + k0 + L)
                if r != q and b > a:
                    lib.lora_unpack(self.tables, plan.chunks_in(r, a, b), a, b, recv[r * L: r * L + b - a])

    def gather_ranges(self, x, ranges):
        """ranges[q] = (a, b): the part of a flat tensor rank q holds, the ranges ascending and covering [0, ranges[-1][1]).  x is this
        rank's part; returns the whole tensor, assembled on every rank (state_dict)."""
        most = max(1, max(b - a for a, b in ranges))
        mine = torch.zeros(most, device=x.device, dtype=x.dtype)
        mine[: x.numel()] = x.reshape(-1)
        every = torch.empty(self.world * most, device=x.device, dtype=x.dtype)
        dist.all_gather_into_tensor(every, mine)
        return torch.cat([every[r * most: r * most + b - a] for r, (a, b) in enumerate(ranges)])
