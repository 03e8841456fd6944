"""GPU check of qfx_gemm_bf16 where its persistent schedule gives each CTA several tiles.

The kernel launches min(total_tiles, SMs) CTAs; CTA c computes tiles c, c + grid, c + 2 grid, ...  Between two tiles of one CTA the
TMA producer runs ahead into the next tile while the consumers run the epilogue, the smem ring's stage / phase carries over, and the
next tile may belong to another problem with another LoRA k-block count.  tools/gemm_tile_check.py never reaches this: each of its
launches has fewer tiles than the H100 has SMs.  Here every launch has more, and is held to:

  (1) schedule invariance, bit for bit: the same operands relaunched as m-slices of at most `SMs` tiles, one problem at a time (every
      CTA then computes exactly one tile), must give identical bits in every output (out, out2, dO_joint and delta, the aliased resid)
      and in every position the launch must not write; the full launch run twice must too.  A tile's k order is fixed by the kernel,
      so no tolerance is involved.  A difference is named by problem, m-tile and n-tile, and by the CTA and the position in that
      CTA's sequence that the kernel's decode and grid rule (restated in `Schedule`) give it;
  (2) gemm_tile_check.run on the same launch (per tile and per row against fp64 scaled by bf16 eager, the rounding rule on the
      kernel's own accumulator, sentinels), with its criteria unchanged.

Launches: the ones a training step makes, recorded from an eager forward + backward of a full-width one-block model built with
bench.py's helpers (`rec_*`), and synthetic ones (tile counts around multiples of the SM count at every block_n and epilogue, K
against the smem ring, six-problem launches that switch LoRA k-block counts, outputs large enough for streamed stores).  Every
launch but the exactly-`SMs` control must give some CTA at least two tiles.

Run stand-alone: `python tools/gemm_sched_check.py [case ...]` (one subprocess per case); tests/test_gemm_schedule.py runs it.
"""
import bisect
import gc
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from harness import ROOT, main  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import gemm_tile_check as gt  # noqa: E402
from gemm_tile_check import (EPI_ADD, EPI_ATTN_DO, EPI_BIAS, EPI_DGELU, EPI_GELU, EPI_NAME, EPI_RESID_GATE, PADC, PADR,  # noqa: E402
                             SENT_F32, _prob, _tile_of, sentinel)
from glue_check import Checks  # noqa: E402

BM = 128
STAGES = {64: 8, 128: 6, 192: 5, 256: 4}  # GemmCfg<BN>::STAGES in gemm.cu
STREAM_BYTES = 48e6                       # outputs larger than this are stored with st.global.cs (gemm.cu: stream_out)
# gemm_tile_check's per-row bound (kernel <= 1.75 x bf16 eager + 5e-4) holds rows of at least this many outputs.  The tile-count
# sweep at block_n 64 has launches of one 64-column n-tile (a prime tile count allows no more) and 17k-51k rows: there the worst
# row ratio over all rows reached 1.78-1.92 (RESID_GATE), 2.0-2.6 (DGELU), 1.84 (GELU) on an H100 while every tile ratio of the
# same launches was <= 0.90, the rounding rule held on the kernel's own accumulator and the launch was bit-identical to its
# one-tile-per-CTA reference.  The per-row ratio of 64 bf16 roundings against 64 others is too noisy at that many rows; at
# N >= 128 it stayed <= 1.70.  Such launches keep every other check and report their row ratio.
ROW_MIN_N = 128


# ============================================================================ the kernel's schedule, restated
def auto_bn(N, epi, block_n=0):
    """the block_n qfx_gemm_bf16 runs for a request (0 = automatic; 1000 + bn = CTA-pair request, run as bn)"""
    bn = block_n - 1000 if block_n >= 1000 else block_n
    if bn == 0 and epi == EPI_ATTN_DO:
        bn = 256 if N % 256 == 0 else 128
    if bn == 0:
        bn = 256 if N % 256 == 0 else 192 if N % 192 == 0 else 128 if N % 128 == 0 else 64
    return bn


def m_tiles(M, bands=None):
    """m-tiles of one problem: dense rows in 128-row tiles, ragged rows two tiles per 256-row band"""
    return 2 * len(bands) if bands is not None else -(-M // BM)


def stream_out(Ms, N, epi):
    return sum(2.0 * M * N * (2 if epi == EPI_GELU else 1) for M in Ms) > STREAM_BYTES


class Schedule:
    """gemm.cu's grid rule and `decode`: tile = n_blk * tiles_m_total + m (m counts the problems' m-tiles in order), grid =
    min(total_tiles, SMs), CTA c computes tiles c, c + grid, ...  So tile t runs on CTA t % grid as that CTA's (t // grid)-th tile."""

    def __init__(self, mtiles, N, bn, sms):
        self.ends = [sum(mtiles[:i + 1]) for i in range(len(mtiles))]
        self.tm, self.tn = self.ends[-1], N // bn
        self.total = self.tm * self.tn
        self.grid = min(self.total, sms)

    def decode(self, tile):
        n_blk, mm = divmod(tile, self.tm)
        prob = bisect.bisect_right(self.ends, mm)
        return prob, mm - (self.ends[prob - 1] if prob else 0), n_blk

    def tile(self, prob, mt, nt):
        return nt * self.tm + (self.ends[prob - 1] if prob else 0) + mt

    def where(self, tile):
        """(CTA, position in its sequence, tiles that CTA runs)"""
        cta = tile % self.grid
        return cta, tile // self.grid, len(range(cta, self.total, self.grid))

    def per_cta(self):
        return self.total // self.grid, -(-self.total // self.grid)

    def stats(self):
        lo, hi = self.per_cta()
        return dict(total_tiles=self.total, grid=self.grid, tiles_per_cta=[lo, hi])


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ============================================================================ (1) schedule invariance
def _bits(t):
    t = t.contiguous()
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _alloc(probs, N, epi, attn, alias, dev):
    """fresh output buffers of one launch: per problem (out, out2) with PADC sentinel columns on each side and PADR rows past M
    (for ATTN_DO `out` is unused and dO_joint / delta are shared); the aliased ADD starts from its resid"""
    bufs = []
    for p in probs:
        M = p["A"].shape[0]
        f = sentinel(M + PADR, N + 2 * PADC, device=dev)
        if alias:
            f[:M, PADC:PADC + N] = p["resid"]
        f2 = sentinel(M + PADR, N + 2 * PADC, device=dev) if (epi == EPI_GELU or p.get("with_out2")) else None
        bufs.append((f, f2))
    dOj = sentinel(attn["B"], attn["H"], attn["S"], 128, device=dev) if epi == EPI_ATTN_DO else None
    delta = torch.full((attn["B"], attn["H"], attn["S"]), SENT_F32, device=dev) if epi == EPI_ATTN_DO else None
    return bufs, dOj, delta


def _problem(L, p, buf, N, epi, alias, dOj, delta, rows=None, bands=None):
    """one gemm_problem over rows [r0, r1) of p (dense) or over the m-tiles of `bands` (ragged)"""
    f, f2 = buf
    M = p["A"].shape[0]
    r0, r1 = rows or (0, M)
    sl = lambda t: None if t is None else t[r0:r1]
    out = f[r0:r1, PADC:PADC + N]
    kw = dict(A2=sl(p.get("A2")), B2=p.get("B2"), kb2=p.get("kb2", 0), a2_col0=p.get("a2_col0", 0), bias=p.get("bias"),
              out2=None if f2 is None else f2[r0:r1, PADC:PADC + N], aux=sl(p.get("aux")),
              row_bands=bands if bands is not None else p.get("bands"))
    if epi in (EPI_RESID_GATE, EPI_ADD):
        kw["resid"] = out if alias else sl(p["resid"])
    if epi == EPI_RESID_GATE:
        rpb = p["rows_per_batch"]
        if r0 % rpb == 0:  # the gate rows of the slice, one per batch as in the full launch
            kw.update(gate=p["gate"][r0 // rpb:], rows_per_batch=rpb)
        else:              # a batch boundary before the slice start: one gate row per output row (same values, same epilogue math)
            kw.update(gate=gt.gate_rows(p, M)[r0:r1].contiguous(), rows_per_batch=1)
    if epi == EPI_ATTN_DO:  # rows [r0, r1) lie inside sample b: its tokens start at joint position s_offset + r0 - b * rpb
        rpb, so = p["rows_per_batch"], p["s_offset"]
        b = r0 // rpb
        assert rows is None or (r1 - 1) // rpb == b, "an ATTN_DO slice must stay inside one sample"
        if rows is None:
            kw.update(rows_per_batch=rpb, s_offset=so)
        else:
            kw.update(rows_per_batch=r1 - r0, s_offset=so + r0 - b * rpb)
            dOj, delta = dOj[b:b + 1], delta[b:b + 1]
        kw["delta"] = delta
        out = dOj
    return L.gemm_problem(sl(p["A"]), p["B"], out, **kw)


def _slices(p, cap_rows, epi):
    """row ranges of the reference launches of one dense problem: at most cap_rows rows each, aligned to the full launch's m-tiles
    where possible; ATTN_DO also cuts at every sample boundary"""
    M = p["A"].shape[0]
    cuts = set(range(0, M, cap_rows)) | {M}
    if epi == EPI_ATTN_DO:
        cuts |= set(range(0, M, p["rows_per_batch"]))
    cuts = sorted(cuts)
    return list(zip(cuts[:-1], cuts[1:]))


def _launch(L, probs, N, K, cfg, sms=None):
    """the full launch (sms None) or its one-tile-per-CTA reference (sms given); returns the output buffers"""
    epi, alias, bn = cfg["epi"], cfg.get("alias", False), cfg["bn"]
    dev = probs[0]["A"].device
    bufs, dOj, delta = _alloc(probs, N, epi, cfg.get("attn"), alias, dev)
    kw = dict(trans_b=cfg["trans_b"], epilogue=epi, alpha=cfg.get("alpha", 1.0), lora_group_n=cfg.get("lora_group_n", 0), block_n=bn)
    if sms is None:
        L.gemm([_problem(L, p, b, N, epi, alias, dOj, delta) for p, b in zip(probs, bufs)], N, K, **kw)
        return bufs, dOj, delta
    per = sms // (N // bn)  # m-tiles per reference launch: each of its tiles gets a CTA of its own
    assert per >= 1, f"N / block_n = {N // bn} n-tiles exceed {sms} SMs: no m-slice runs one tile per CTA"
    for p, b in zip(probs, bufs):
        bands = p.get("bands")
        if bands is None:
            for r in _slices(p, per * BM, epi):
                L.gemm([_problem(L, p, b, N, epi, alias, dOj, delta, rows=r)], N, K, **kw)
            continue
        from qflux_b200 import lib
        nb = per // 2  # bands per reference launch (two m-tiles each); each sub-list zero-fills the same dead rows
        assert nb >= 1, f"a band's two m-tiles times {N // bn} n-tiles exceed {sms} SMs"
        for i in range(0, len(bands.host_tiles), nb):
            sub = lib.RowBands(bands.host_tiles[i:i + nb], bands.host_dead, dev)
            L.gemm([_problem(L, p, b, N, epi, alias, dOj, delta, bands=sub)], N, K, **kw)
    return bufs, dOj, delta


def _views(probs, N, epi, out):
    """per problem {name: (token-major [M, C] view, columns per n-tile unit)} of one launch's outputs, and the positions outside them"""
    bufs, dOj, delta = out
    views, outside = [], []
    covered = torch.zeros(dOj.shape[2], dtype=torch.bool, device=dOj.device) if epi == EPI_ATTN_DO else None
    for p, (f, f2) in zip(probs, bufs):
        M = p["A"].shape[0]
        v = {}
        if epi == EPI_ATTN_DO:
            rpb, so = p["rows_per_batch"], p["s_offset"]
            nb = M // rpb
            v["dO_joint"] = (dOj[:nb, :, so:so + rpb].permute(0, 2, 1, 3).reshape(M, N), 1)
            v["delta"] = (delta[:nb, :, so:so + rpb].permute(0, 2, 1).reshape(M, -1), 128)
            covered[so:so + rpb] = True
        else:
            v["out"] = (f[:M, PADC:PADC + N], 1)
        for name, buf in (("out", f if epi != EPI_ATTN_DO else None), ("out2", f2)):
            if buf is None:
                continue
            if name == "out2":
                v["out2"] = (buf[:M, PADC:PADC + N], 1)
            inner = torch.zeros_like(buf, dtype=torch.bool)
            inner[:M, PADC:PADC + N] = True
            outside.append((f"p{len(views)}_{name} outside its rows / column slice", buf[~inner]))
        views.append(v)
    if epi == EPI_ATTN_DO:
        outside += [("dO_joint at uncovered joint positions", dOj[:, :, ~covered]), ("delta at uncovered joint positions", delta[:, :, ~covered])]
    return views, outside


def compare(c, tag, probs, N, cfg, a, b, sched, what):
    """bitwise a == b over every output of one launch; each differing tile is named with its CTA and position; returns the list of
    differing (problem, m-tile, n-tile, CTA, position)"""
    va, oa = _views(probs, N, cfg["epi"], a)
    vb, ob = _views(probs, N, cfg["epi"], b)
    bad = {}
    for i, p in enumerate(probs):
        M = p["A"].shape[0]
        tile_of, _ = _tile_of(M, p.get("bands"), p["A"].device)
        for name, (x, unit) in va[i].items():
            y = vb[i][name][0]
            d = (_bits(x) != _bits(y))
            if not bool(d.any()):
                continue
            r, col = d.nonzero(as_tuple=True)
            mt = tile_of[r]
            nt = (col * unit) // cfg["bn"]
            for key, n in zip(*torch.unique(torch.stack([mt, nt], 1), dim=0, return_counts=True)):
                k = (i, int(key[0]), int(key[1]))
                e = bad.setdefault(k, [0, set()])
                e[0] += int(n)
                e[1].add(name)
    found = []
    for (i, mt, nt), (n, names) in sorted(bad.items()):
        cta, pos, runs = sched.where(sched.tile(i, mt, nt))
        found.append((i, mt, nt, cta, pos))
        if len(found) <= 8:
            c.fail.append(f"{tag} {what}: problem {i} m-tile {mt} n-tile {nt} ({'/'.join(sorted(names))}, {n} elements) differs; "
                          f"CTA {cta} computes it as tile {pos} of its {runs}")
    if len(found) > 8:
        c.fail.append(f"{tag} {what}: {len(found)} tiles differ in all, at positions {sorted({f[4] for f in found})}")
    for (name, x), (_, y) in zip(oa, ob):
        if not bool((_bits(x) == _bits(y)).all()):
            c.fail.append(f"{tag} {what}: {name} differs")
            found.append(("outside", name))
    return found


def invariance(c, tag, probs, N, K, cfg, sms, L=None):
    """(1): the full launch against its one-tile-per-CTA reference and against itself run again"""
    from qflux_b200 import lib
    L = L or lib
    sched = Schedule([m_tiles(p["A"].shape[0], p.get("bands") and p["bands"].host_tiles) for p in probs], N, cfg["bn"], sms)
    full = _launch(L, probs, N, K, cfg)
    again = _launch(L, probs, N, K, cfg)
    ref = _launch(L, probs, N, K, cfg, sms=sms)
    bad = compare(c, tag, probs, N, cfg, full, ref, sched, "full launch vs one tile per CTA")
    rep = compare(c, tag, probs, N, cfg, full, again, sched, "full launch run twice")
    c.res[f"{tag}_bad_tiles"] = [list(t) for t in bad]
    c.res[f"{tag}_repeat_bad_tiles"] = [list(t) for t in rep]
    return sched


# ============================================================================ one launch, both checks
def check(c, tag, probs, N, K, cfg, sms, fp64=True, control=False):
    """(1) and (2) on one launch; cfg: epi, trans_b, bn, [alpha, lora_group_n, attn, alias].  Records the schedule and fails a launch
    (other than the exactly-SMs control) on which no CTA gets two tiles."""
    t0 = time.time()
    if probs[0]["A"].is_cuda:
        torch.cuda.reset_peak_memory_stats()
    sched = invariance(c, tag, probs, N, K, cfg, sms)
    if fp64:
        gt.run(c, tag, probs, N, K, trans_b=cfg["trans_b"], epi=cfg["epi"], alpha=cfg.get("alpha", 1.0), bn=cfg["bn"],
               lora_group_n=cfg.get("lora_group_n", 0), attn=cfg.get("attn"), emu_check=False, alias=cfg.get("alias", False),
               rows=N >= ROW_MIN_N)
    st = dict(sched.stats(), stream_out=stream_out([p["A"].shape[0] for p in probs], N, cfg["epi"]), N=N, K=K, bn=cfg["bn"],
              epi=EPI_NAME[cfg["epi"]], seconds=round(time.time() - t0, 2))
    ratios = lambda suf: max((v for k, v in c.res.items() if k.startswith(tag + "_p") and k.endswith(suf)), default=None)
    st.update(tile_ratio_max=ratios("_tile_ratio_max"), row_ratio_max=ratios("_row_ratio_max"))
    if probs[0]["A"].is_cuda:
        st["peak_gb"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
    c.res[f"{tag}_sched"] = st
    if not control and st["tiles_per_cta"][1] < 2:
        c.fail.append(f"{tag}: no CTA computes two tiles ({sched.total} tiles on {sched.grid} CTAs): not a multi-tile check")
    return st


# ============================================================================ synthetic launches (plans are pure arithmetic)
EPI_SETS = [(EPI_BIAS, False), (EPI_BIAS, True), (EPI_GELU, False), (EPI_RESID_GATE, False), (EPI_DGELU, True), (EPI_ADD, True),
            (EPI_ATTN_DO, True)]


def _epi_tag(epi, trans_b):
    return f"{EPI_NAME[epi]}_{'nn' if trans_b else 'nt'}"


def bns(epi):
    return (128, 256) if epi == EPI_ATTN_DO else (64, 128, 192, 256)


def tile_counts(sms):
    return (sms, sms + 1, 2 * sms - 1, 2 * sms + 1, 3 * sms + 7)


def _spec(epi, trans_b, bn, mts, tn, K, *, kb2=(1,), seed=1, alias=False, lora_group_n=0, rpb=97, shift=1.5):
    """a launch plan: problems with mts[i] m-tiles (the last tile of each partly filled), N = tn * bn"""
    probs = []
    for i, mt in enumerate(mts):
        if epi == EPI_ATTN_DO:
            r = 64 * mt - 18 - 3 * i  # two samples per problem: 2 r rows fill mt tiles
            M = 2 * r
        else:
            M, r = BM * mt - 37 + 9 * (i % 3), rpb
        k2 = kb2[i % len(kb2)]
        probs.append(dict(M=M, kb2=k2, a2_col0=64 if k2 else 0, groups=(tn * bn) // lora_group_n if lora_group_n else 1,
                          bias=not trans_b, rows_per_batch=r, with_out2=epi in (EPI_RESID_GATE, EPI_ATTN_DO) and i % 2 == 0,
                          shift=shift * i, seed=seed + 10 * i))
    spec = dict(epi=epi, trans_b=trans_b, bn=bn, N=tn * bn, K=K, probs=probs, lora_group_n=lora_group_n, alias=alias,
                alpha=1.0 if epi in (EPI_GELU, EPI_RESID_GATE) else 0.5)
    if epi == EPI_ATTN_DO:
        so = 5
        for p in probs:
            p["s_offset"], so = so, so + p["rows_per_batch"]
        spec["attn"] = dict(B=2, H=tn * bn // 128, S=so + 3)  # positions [0, 5) and the last 3 stay uncovered
    return spec


def plan(sms):
    """{case: [(tag, spec, control)]} of the synthetic launches for a card with `sms` SMs"""
    cases = {}
    for epi, tb in EPI_SETS:  # tile counts around multiples of the SM count, at every block_n
        out = []
        for bn in bns(epi):
            for j, T in enumerate(tile_counts(sms)):
                tn = next(d for d in (4, 3, 2, 1) if T % d == 0)
                s = _spec(epi, tb, bn, [T // tn], tn, 128, alias=epi == EPI_ADD and j % 2 == 1, seed=T)
                out.append((f"bn{bn}_T{T}", s, T == sms))
        cases[f"tiles_{_epi_tag(epi, tb)}"] = out
    for bn in (64, 128, 192, 256):  # K against the smem ring: one k-block (the producer runs STAGES tiles ahead), a full ring, one more
        S, T = STAGES[bn], 2 * sms + 1
        out = []
        for K in (64, S * 64, S * 64 + 64, 4096):
            for tb in (False, True):
                out.append((f"K{K}_{'nn' if tb else 'nt'}", _spec(EPI_BIAS, tb, bn, [T], 1, K, kb2=(0,), seed=K), False))
        cases[f"ring_bn{bn}"] = out
    for epi, tb in EPI_SETS:  # six problems whose LoRA k-block counts alternate: a CTA's next tile changes problem and k-block count
        bn, tn = (256, 1) if epi == EPI_ATTN_DO else (128, 3)
        tm = -(-(2 * sms + 7) // tn)
        w = (0.05, 0.3, 0.1, 0.25, 0.02, 0.28)
        mts = [max(1, round(tm * x)) for x in w]
        mts[-1] += max(0, tm - sum(mts))
        s = _spec(epi, tb, bn, mts, tn, 192, kb2=(0, 2, 1, 3, 0, 2), lora_group_n=bn if not tb else 0, shift=1.5)
        cases.setdefault("switch", []).append((_epi_tag(epi, tb), s, False))
    for epi, tb in EPI_SETS:  # outputs past 48 MB: the stores stream past L2
        mt = 96
        s = _spec(epi, tb, 256, [mt], 8, 128, alias=epi == EPI_ADD, rpb=1000)
        cases.setdefault("stream", []).append((_epi_tag(epi, tb), s, False))
    return cases


def build_probs(spec, dev):
    """fresh seeded operands of a plan (gemm_tile_check._prob: contiguous, each problem's epilogue operands shifted apart)"""
    from qflux_b200 import lib
    N, K, epi, tb = spec["N"], spec["K"], spec["epi"], spec["trans_b"]
    probs = []
    for g in spec["probs"]:
        p = _prob(g["M"], N, K, tb, g["seed"], kb2=g["kb2"], a2_col0=g["a2_col0"], groups=g["groups"], bias=g["bias"], epi=epi,
                  rows_per_batch=g["rows_per_batch"] if epi == EPI_RESID_GATE else 0, with_out2=g["with_out2"], shift=g["shift"],
                  device=dev)
        if epi == EPI_ATTN_DO:
            p.update(rows_per_batch=g["rows_per_batch"], s_offset=g["s_offset"])
        if g.get("bands"):
            p["bands"] = lib.RowBands(list(g["bands"][0]), [list(d) for d in g["bands"][1]], dev)
        probs.append(p)
    return probs


def _cfg(spec):
    return {k: spec[k] for k in ("epi", "trans_b", "bn", "alpha", "lora_group_n", "alias") if k in spec} | (
        dict(attn=spec["attn"]) if spec.get("attn") else {})


def run_planned(name):
    c = Checks()
    sms = num_sms()
    t0 = time.time()
    for tag, spec, control in plan(sms)[name]:
        probs = build_probs(spec, "cuda")
        check(c, tag, probs, spec["N"], spec["K"], _cfg(spec), sms, control=control)
        del probs
    c.res.update(sms=sms, seconds=round(time.time() - t0, 1))
    return _summary(c)


def _summary(c):
    """the case's result with the per-launch schedule lines first; fp64 detail stays in the dict"""
    out = c.out()
    sched = {k[:-6]: v for k, v in out.items() if k.endswith("_sched")}
    for k in list(out):
        if k.endswith("_sched"):
            del out[k]
    if torch.cuda.is_available():
        torch.cuda.empty_cache()
    return dict(launches=sched, **out)


# ============================================================================ the training step's own launches
SITE_KINDS = ("qkv", "out_resid_gate", "down_resid_gate", "s_out", "mlp_up_gelu", "dgelu", "attn_do", "lora_u", "lora_t",
              "proj_out_fwd", "proj_out_dgrad", "add_alias")


def site_kind(rec, D, C_out, rp):
    """which call site of the step a recorded launch is, from its geometry (D = model width)"""
    N, K, epi, tb = rec["N"], rec["K"], rec["epi"], rec["trans_b"]
    if epi == EPI_ATTN_DO:
        return "attn_do"
    if epi == EPI_DGELU:
        return "dgelu"
    if epi == EPI_GELU:
        return "mlp_up_gelu" if N == 4 * D and K == D else "gelu"
    if epi == EPI_RESID_GATE:
        return {D: "out_resid_gate", 4 * D: "down_resid_gate", 5 * D: "s_out"}.get(K, "resid_gate") if N == D else "resid_gate"
    if epi == EPI_ADD:
        return "add_alias" if all(p["alias"] for p in rec["probs"]) else "add"
    if tb and N == rp:
        return "lora_u"
    if not tb and N == C_out and K == D and all(p["bias"] for p in rec["probs"]):  # a LoRA projection at N = C_out has no bias
        return "proj_out_fwd"
    if tb and N == D and K == C_out:
        return "proj_out_dgrad"
    if not tb and N == 3 * D and rec["lora_group_n"] == D:
        return "qkv"
    if not tb and N % rp == 0 and N < D:
        return "lora_t"
    return "bias_nt" if not tb else "bias_nn"


class Recorder:
    """wraps lib.gemm_problem / lib.gemm: every launch's geometry (per problem: M, kb2, a2_col0, A2 width, rows_per_batch, s_offset,
    row bands, which epilogue operands are present, resid aliasing out; per launch: N, K, trans_b, epilogue, alpha, lora_group_n and
    the block_n the kernel runs)"""

    def __init__(self, lib):
        self.lib, self.launches = lib, []

    def __enter__(self):
        lib = self.lib
        self._saved = (lib.gemm_problem, lib.gemm)
        gp, gm = self._saved

        def gemm_problem(A, B, out, **kw):
            p = gp(A, B, out, **kw)
            rb, d, r = kw.get("row_bands"), kw.get("delta"), kw.get("resid")
            p._geom = dict(M=A.shape[0], kb2=kw.get("kb2", 0), a2_col0=kw.get("a2_col0", 0), rows_per_batch=kw.get("rows_per_batch", 0),
                           s_offset=kw.get("s_offset", 0), bias=kw.get("bias") is not None, out2=kw.get("out2") is not None,
                           resid=r is not None, gate=kw.get("gate") is not None, aux=kw.get("aux") is not None,
                           alias=r is not None and r.data_ptr() == out.data_ptr(),
                           bands=None if rb is None else (tuple(rb.host_tiles), tuple(tuple(x) for x in rb.host_dead)),
                           attn=tuple(out.shape[:3]) if d is not None else None)
            return p

        def gemm(problems, N, K, *, trans_b=False, epilogue=EPI_BIAS, alpha=1.0, lora_group_n=0, block_n=0):
            self.launches.append(dict(N=N, K=K, trans_b=bool(trans_b), epi=epilogue, alpha=float(alpha), lora_group_n=lora_group_n,
                                      bn=auto_bn(N, epilogue, block_n), probs=[dict(p._geom) for p in problems]))
            return gm(problems, N, K, trans_b=trans_b, epilogue=epilogue, alpha=alpha, lora_group_n=lora_group_n, block_n=block_n)

        lib.gemm_problem, lib.gemm = gemm_problem, gemm
        return self

    def __exit__(self, *exc):
        self.lib.gemm_problem, self.lib.gemm = self._saved


RECORDED = {  # case: (bench config, B)
    "rec_qwen_edit_b1": ("qwen_edit", 1),
    "rec_qwen_plus_b1": ("qwen_plus_sharded", 1),
    "rec_qwen_multires_b2": ("qwen_multires", 2),
    "rec_qwen_edit_b4": ("qwen_edit", 4),
    "rec_flux_kontext_b2": ("flux_kontext", 2),
}


def record(config, B, dev, tiny=None, cfg_update=None):
    """one eager forward + backward of bench.py's model of `config` at one block (FLUX: one double + one single block), full width
    unless `tiny` (depth_check.build's reduced model); returns (launches, D, C_out, lora_rp)"""
    import bench
    import depth_check as dc
    from qflux_b200 import lib
    from qflux_b200.train_step import FluxKontextStep, QwenImageEditStep
    cfg = dict(bench.CONFIGS[config], B=B, **(cfg_update or {}))
    qwen = cfg["model"] == "qwen"
    torch.manual_seed(1234)
    if tiny is not None:
        m = dc.build(cfg, dev, dict(tiny, layers=1, single=1))
    else:
        m = bench.build_model(dev, 1, cfg) if qwen else bench.build_flux(dev, cfg, 0.01)
    emb = bench.make_batch(cfg, config, host=False)
    L = emb["image_latents"].shape[1]
    noise = torch.randn(B, L, 64, generator=torch.Generator().manual_seed(7)).bfloat16()
    kw = dict(noise=noise, u=torch.tensor(dc.U[:B])) if qwen else dict(noise=noise, t=torch.tensor(dc.T_FLUX[:B]))
    Step = QwenImageEditStep if qwen else FluxKontextStep
    with Recorder(lib) as rec:
        Step(m, "attention_mask" if config == "qwen_multires" else "mse", max_grad_norm=0.0, use_cuda_graph=False).train_step(emb, **kw)
    if dev.type == "cuda":
        torch.cuda.synchronize()
    out = (rec.launches, m.D, m.C_out, m.lora_rp)
    del m
    gc.collect()
    return out


def _key(rec):
    return repr({k: v for k, v in rec.items()})


def replay_spec(rec, seed):
    """a recorded launch rebuilt as a plan on fresh operands"""
    N, lgn = rec["N"], rec["lora_group_n"]
    probs = []
    for i, g in enumerate(rec["probs"]):
        probs.append(dict(M=g["M"], kb2=g["kb2"], a2_col0=g["a2_col0"], groups=N // lgn if lgn else 1, bias=g["bias"],
                          rows_per_batch=g["rows_per_batch"] or g["M"], with_out2=g["out2"] and rec["epi"] != EPI_GELU,
                          shift=1.5 * i, seed=seed + 10 * i, s_offset=g["s_offset"], bands=g["bands"]))
    spec = dict(epi=rec["epi"], trans_b=rec["trans_b"], bn=rec["bn"], N=N, K=rec["K"], probs=probs, lora_group_n=lgn,
                alias=all(g["alias"] for g in rec["probs"]), alpha=rec["alpha"])
    a = rec["probs"][0]["attn"]
    if a is not None:
        spec["attn"] = dict(B=a[0], H=a[1], S=a[2])
    return spec


def run_recorded(name, dev="cuda", tiny=None, cfg_update=None, sms=None, fp64=True):
    """(2) + (1) on every distinct launch of one recorded step; each epilogue present must have a launch with >= 2 tiles on a CTA"""
    c = Checks()
    t0 = time.time()
    config, B = RECORDED[name]
    launches, D, C_out, rp = record(config, B, torch.device(dev), tiny, cfg_update)
    sms = sms or num_sms()
    seen, kinds = {}, {}
    for rec in launches:
        seen.setdefault(_key(rec), rec)
    for j, rec in enumerate(seen.values()):
        kind = site_kind(rec, D, C_out, rp)
        tag = f"{kind}_{j}"
        spec = replay_spec(rec, 100 * j + 1)
        probs = build_probs(spec, dev)
        cfg = _cfg(spec)
        st = check(c, tag, probs, spec["N"], spec["K"], cfg, sms, fp64=fp64, control=True)
        st.update(kind=kind, Ms=[p["M"] for p in spec["probs"]], kb2=[p["kb2"] for p in spec["probs"]],
                  s_offset=[p["s_offset"] for p in spec["probs"]] if rec["epi"] == EPI_ATTN_DO else None)
        kinds.setdefault(kind, []).append(tag)
        del probs
    best = {}
    for k, v in c.res.items():
        if k.endswith("_sched"):
            best[v["epi"]] = max(best.get(v["epi"], 0), v["tiles_per_cta"][1])
    for e, hi in best.items():
        if hi < 2:
            c.fail.append(f"{name}: no recorded {e} launch gives a CTA two tiles")
    c.res.update(sms=sms, launches_recorded=len(launches), distinct=len(seen), kinds=kinds, max_tiles_per_cta_by_epilogue=best,
                 seconds=round(time.time() - t0, 1))
    return _summary(c)


CASES = {}
for _n in ("tiles_" + _epi_tag(e, t) for e, t in EPI_SETS):
    CASES[_n] = (lambda n: lambda: run_planned(n))(_n)
for _n in ("ring_bn64", "ring_bn128", "ring_bn192", "ring_bn256", "switch", "stream"):
    CASES[_n] = (lambda n: lambda: run_planned(n))(_n)
for _n in RECORDED:
    CASES[_n] = (lambda n: lambda: run_recorded(n))(_n)

if __name__ == "__main__":
    main(CASES, os.path.abspath(__file__), "gemm_sched_check.log", timeout=900)
