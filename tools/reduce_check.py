"""GPU check of the backward's fp32 reductions and the conditioning GEMV, per element against fp64 references computed on the device
from the exact bf16 inputs:

  qfx_lora_wgrad_tc (+ _det)  every LoRA dA / dB except the 64-channel embedder's (wgmma, rows split over CTAs);
  qfx_lora_wgrad (+ _det)     the CUDA-core path of that embedder;
  qfx_mod_grad (+ _det)       the AdaLN shift / scale / gate gradients, in the model's three call forms;
  qfx_flow_loss (+ _det)      the flow-matching loss and dpred;
  qfx_gemv_act                every modulation vector and the timestep MLP of the forward.

Every accumulated output is pre-filled with non-zero values and compared with `init + ref`; every output sits in a larger buffer whose
other elements (before, after and between tensors, untouched columns of [B, 6D] views, columns past N) hold a sentinel that must come
back bit for bit.  Each case runs the atomic entry point and its `_det` twin against the same bound, the twin with a NaN-filled scratch
of exactly lib.det_scratch_*, twice (the two results must be bit-identical).

The atomic wgrad_tc and mod_grad choose their row splits from the SM count; `wgrad_tc_plan` / `mod_grad_plan` restate the host formulas
and the `*_edges` cases derive shapes from the card's SM count at which the last split holds one row or exactly one k-block, the row
count is a multiple of 64, or it is one more / one less than rows x splits.  Each case reports its plan.

Bounds (per element):
  reductions   |out - (init + ref)| <= RED_TOL * (|init| + sum |terms|)  (+ the flip term of a bf16-rounded operand, where one is formed)
  flow dpred   bit for bit an fp32 restatement in the kernel's order, bf16((((2 norm) w) d) grad_scale), and within one bf16 ulp of fp64
  gemv_act     RED_TOL * sum |terms| + the SiLU flip term + the output rounding
Run stand-alone: `python tools/reduce_check.py [case ...]` (one subprocess per case).
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from harness import ROOT, main  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from glue_check import RED_TOL, Checks, _mk, _up, ulp_bf16  # noqa: E402,F401

BF, F32, F64 = torch.bfloat16, torch.float32, torch.float64
SENT = -0.01171875   # fp32 sentinel: small, so that any add into it changes its bits
SENT_BF = -7.25      # bf16 sentinel
BIG = 4096.0         # B's columns j >= r of each group: a slip in the column mapping shows
GAP = 5              # sentinel elements before, between and after the tensors of a flat buffer


def _cdiv(a, b):
    return -(-a // b)


# ============================================================================ split plans (the host formulas, restated)
def wgrad_tc_plan(M, Na, sms):
    """qfx_lora_wgrad_tc: splits = min(ceil(2 SMs / tiles), ceil(M / 256)), rows rounded up to 64; the grid has ceil(M / rows) splits"""
    cap = _cdiv(2 * sms, Na // 128)
    splits = max(1, min(cap, _cdiv(M, 256)))
    rows = _cdiv(_cdiv(M, splits), 64) * 64
    n = _cdiv(M, rows)
    return dict(M=M, splits=splits, rows=rows, grid_splits=n, last=M - rows * (n - 1), sm_bound=cap < _cdiv(M, 256))


def mod_grad_plan(rpb, B, D, sms):
    """qfx_mod_grad: splits = min(ceil(4 SMs / (cb B)), ceil(rpb / 32)), cb = ceil(D / 256); split z holds rows [z per, (z+1) per)"""
    cap = _cdiv(4 * sms, _cdiv(D, 256) * B)
    splits = max(1, min(cap, _cdiv(rpb, 32)))
    per = _cdiv(rpb, splits)
    n = _cdiv(rpb, per)  # splits that hold rows (the rest, if any, contribute zeros)
    return dict(rows_per_batch=rpb, splits=splits, rows=per, grid_splits=n, last=rpb - per * (n - 1), sm_bound=cap < _cdiv(rpb, 32))


def split_edges(plan, lo, hi, unit):
    """The first value in [lo, hi) for each split edge among those whose split count the SM count sets: the last split holds one
    row; it holds exactly one k-block of `unit` rows; a multiple of 64 with a partial last split; and v = rows * splits - 1 / + 1
    around the first exact fill.  (An edge can be out of reach: with S SM-set splits of mod_grad, rows > 32 S, so every split
    holds more than 32 rows and the last one at least rows - S + 1; one row then needs S >= 33.)"""
    found = {}
    for v in range(lo, hi):
        p = plan(v)
        if p["grid_splits"] < 2 or not p["sm_bound"]:
            continue
        if p["last"] == 1:
            found.setdefault("last_one_row", v)
        if p["last"] == unit:
            found.setdefault("last_one_kblock", v)
        if v % 64 == 0 and p["last"] != p["rows"] and v not in found.values():
            found.setdefault("mult64", v)
        if v == p["rows"] * p["grid_splits"] and "fill_minus1" not in found:
            found["fill_minus1"], found["fill_plus1"] = v - 1, v + 1
        if len(found) == 5:
            break
    return found


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ============================================================================ fp64 references (device-agnostic; checked on CPU too)
def wgrad_tc_ref(A, B, r, G, mode=0, Dg=0):
    """per group g: (sum_m A[m, i] B[m, g*64 + j], sum_m |A B|) for the group's A columns, j < r, in fp64"""
    Ad, Bd = A.double(), B.double()
    out = []
    for g in range(G):
        a = Ad[:, g * Dg:(g + 1) * Dg] if mode == 1 else Ad
        b = Bd[:, g * 64:g * 64 + r]
        out.append((a.t() @ b, a.abs().t() @ b.abs()))
    return out


def lora_wgrad_ref(P, Q, r):
    Pd, Qd = P.double(), Q.double()[:, :r]
    return Pd.t() @ Qd, Pd.abs().t() @ Qd.abs()


def mod_m(m, mean=None, rstd=None):
    """the operand the product reduction multiplies g with: m' = bf16((m - mean) rstd) from the fp32 statistics, else m"""
    if mean is None:
        return m
    return ((m.float() - mean[:, None]) * rstd[:, None]).to(BF)


def mod_grad_ref(g, rpb, m=None, mean=None, rstd=None):
    """fp64 column sums per sample: sum (sum_t g, sum_t |g|); with m: prod, its magnitude, and with row statistics the flip term
    sum_t |g| ulp(m') of the bf16-rounded m' (the kernel rounds the same fp32 value, but a fast-math build may land on its neighbour)"""
    D = g.shape[1]
    gd = g.double().view(-1, rpb, D)
    out = dict(sum=gd.sum(1), sum_mag=gd.abs().sum(1))
    if m is not None:
        md = mod_m(m, mean, rstd).double().view(-1, rpb, D)
        out["prod"], out["prod_mag"] = (gd * md).sum(1), (gd * md).abs().sum(1)
        out["flip"] = (gd.abs() * _up(md)).sum(1) if mean is not None else torch.zeros_like(out["prod"])
    return out


def flow_loss_ref(pred, x0, noise, w, norm, grad_scale):
    """(loss in fp64, norm * sum |w d^2|, dpred by the kernel's fp32 rule, dpred in fp64); d = pred - bf16(noise - x0), the scalars
    as the fp32 values the C ABI receives"""
    B, L, C = x0.shape
    dev = pred.device
    n32, gs32 = torch.tensor(norm, dtype=F32, device=dev), torch.tensor(grad_scale, dtype=F32, device=dev)
    tgt = (noise.float() - x0.float()).to(BF)
    d32 = pred[:, :L].float() - tgt.float()
    w32 = w.float()[..., None] if w is not None else torch.ones(B, L, 1, device=dev)
    rule = torch.zeros(pred.shape, dtype=BF, device=dev)
    rule[:, :L] = ((((2 * n32) * w32) * d32) * gs32).to(BF)
    d64, w64 = pred[:, :L].double() - tgt.double(), w32.double()
    terms = w64 * d64 * d64
    dp64 = torch.zeros(pred.shape, dtype=F64, device=dev)
    dp64[:, :L] = 2 * n32.double() * w64 * d64 * gs32.double()
    return n32.double() * terms.sum(), n32.double() * terms.abs().sum(), rule, dp64


def gemv_ref(x, W, bias, act):
    """(y in fp64, sum |terms|, flip term): y = act(x) W^T + bias with act(x) = bf16(SiLU(x)) as the kernel (and eager) rounds it; the
    kernel's fast-math SiLU may land on the neighbouring bf16 value, which moves y by at most ulp(act(x)) |W| per term"""
    xin = F.silu(x.float()).to(BF).double() if act == 1 else x.double()
    Wd = W.double()
    y = xin @ Wd.t()
    mag = xin.abs() @ Wd.abs().t()
    if bias is not None:
        y, mag = y + bias.double(), mag + bias.double().abs()
    flip = _up(xin) @ Wd.abs().t() if act == 1 else torch.zeros_like(y)
    return y, mag, flip


# ============================================================================ buffers with sentinels
class Slots:
    """fp32 tensors at offsets in one flat buffer, with SENT before, between and after them"""

    def __init__(self, sizes, device="cuda"):
        self.offs, o = [], GAP
        for n in sizes:
            self.offs.append(o)
            o += n + GAP
        self.sizes = sizes
        self.buf = torch.full((o,), SENT, device=device)
        self.free = torch.ones(o, dtype=torch.bool, device=device)
        for off, n in zip(self.offs, sizes):
            self.free[off:off + n] = False

    def __getitem__(self, k):
        return self.buf[self.offs[k]:self.offs[k] + self.sizes[k]]


def _bits(t):
    return t.view(torch.int32) if t.dtype == F32 else t.view(torch.int16)


def _sentinels(c, name, buf, free, value):
    bad = int((_bits(buf)[free] != _bits(torch.full((1,), value, dtype=buf.dtype, device=buf.device))).sum())
    c.check(bad == 0, f"{name}: {bad} sentinel elements changed")


def _worst(c, key, v):
    c.res[key] = max(c.res.get(key, 0.0), float(v))


def _bound(c, key, name, got, want, bound):
    """|got - want| <= bound element-wise (fp64); records the worst error / bound under `key`"""
    d = (got.double() - want).abs()
    ratio = (d / bound.clamp_min(1e-300)).max().item() if d.numel() else 0.0
    _worst(c, key, ratio)
    c.check(bool((d <= bound).all()), f"{name}: {int((d > bound).sum())} elements beyond the bound (worst {ratio:.3g})")


def _init(n, seed, scale=4.0):
    """non-zero accumulator contents"""
    v = _mk(n, seed=seed, dtype=F32) * scale
    return torch.where(v == 0, torch.full_like(v, 0.5), v)


def _run_both(c, tag, atomic, det, scratch_floats, outputs, check):
    """atomic(slots) and det(slots, scratch) into freshly initialised copies of `outputs` (Slots factory); det twice, bit-identical"""
    res = {}
    for var in ("atomic", "det", "det_repeat"):
        s = outputs()
        if var == "atomic":
            atomic(s)
        else:
            scr = torch.full((scratch_floats,), float("nan"), device="cuda")
            det(s, scr)
        res[var] = s
    torch.cuda.synchronize()
    for var in ("atomic", "det"):
        check(var, res[var])
    same = torch.equal(_bits(res["det"].buf), _bits(res["det_repeat"].buf))
    c.check(same, f"{tag}: det twin differs between two launches")


# ============================================================================ qfx_lora_wgrad_tc
WG_M = [1, 63, 64, 65, 256, 257, 1408, 8192]  # 1408 / 8192: Qwen-Image-Edit's per-stream rows at B = 4
WG_R = [1, 4, 7, 16, 33, 64]
WG_NA = [128, 384, 3072, 12288]


def _wgrad_tc_one(c, mode, G, Dg, r, Na, M, layout, seed):
    from qflux_b200 import lib
    tag = f"wgrad_tc mode{mode} G{G} r{r} Na{Na} M{M} {layout}"
    A = _mk(M, Na + 72, seed=seed)[:, 8:8 + Na]                       # lda = Na + 72, base 16 bytes into the row
    Bm = _mk(M, 64 * G + 24, seed=seed + 1)[:, 8:8 + 64 * G]             # ldb = 64 G + 24
    for g in range(G):
        Bm[:, g * 64 + r:(g + 1) * 64] = BIG
    rows = Dg if mode == 1 else Na
    gs_i, gs_j = (r, 1) if layout == "dB" else (1, rows)                # dB [out, r] / dA [r, in]
    refs = wgrad_tc_ref(A, Bm, r, G, mode, Dg)
    inits = [_init(rows * r, seed + 10 + g) for g in range(G)]

    def outputs():
        s = Slots([rows * r] * G)
        for g in range(G):
            s[g].copy_(inits[g])
        return s

    def view(t):
        return torch.as_strided(t, (rows, r), (gs_i, gs_j))

    def check(var, s):
        for g, (ref, mag) in enumerate(refs):
            i0 = view(inits[g]).double()
            _bound(c, f"wgrad_tc_{var}_max_err_over_bound", f"{tag} {var} group {g}", view(s[g]), i0 + ref, RED_TOL * (i0.abs() + mag))
        _sentinels(c, f"{tag} {var}", s.buf, s.free, SENT)

    ng = 1 if mode == 1 else G
    _run_both(c, tag, lambda s: lib.lora_wgrad_tc(A, Bm, [s[g] for g in range(G)], gs_i, gs_j, r, mode=mode, Dg=Dg),
              lambda s, scr: lib.lora_wgrad_tc_det(A, Bm, [s[g] for g in range(G)], gs_i, gs_j, r, mode=mode, Dg=Dg, scratch=scr),
              lib.det_scratch_wgrad_tc(M, Na, ng, r), outputs, check)


def wgrad_tc_sweep(mode, G, Dg=0):
    c = Checks()
    sms = num_sms()
    if mode == 0:
        triples = [(WG_R[k % 6], WG_NA[(k + G) % 4], M) for k, M in enumerate(WG_M)] + [(64, 12288, 8192), (7, 3072, 1408)]
    else:
        triples = [(r, G * Dg, M) for r, M in zip([33, 7, 64, 1, 16], [1, 65, 257, 1408, 8192])]
    c.res["plans"] = []
    for k, (r, Na, M) in enumerate(triples):
        c.res["plans"].append(dict(wgrad_tc_plan(M, Na, sms), r=r, Na=Na))
        _wgrad_tc_one(c, mode, G, Dg, r, Na, M, ("dB", "dA")[k % 2], seed=100 * k + 7)
    c.res["sms"] = sms
    return c.out()


def wgrad_tc_edges(Na, G=2):
    """M at the atomic kernel's SM-derived split edges (and the det twin at the same M)"""
    c = Checks()
    sms = num_sms()
    edges = split_edges(lambda M: wgrad_tc_plan(M, Na, sms), 257, 1 << 18, 64)
    c.res["sms"], c.res["edges"] = sms, edges
    c.check(len(edges) == 5, f"split edges not all found: {sorted(edges)}")
    c.res["plans"] = {}
    for k, (name, M) in enumerate(sorted(edges.items())):
        r = (16, 7, 33, 64, 1)[k % 5]
        c.res["plans"][name] = dict(wgrad_tc_plan(M, Na, sms), r=r)
        _wgrad_tc_one(c, 0, G, 0, r, Na, M, ("dB", "dA")[k % 2], seed=300 + k)
    return c.out()


# ============================================================================ qfx_lora_wgrad (CUDA cores)
LW_DP = [64, 100, 128, 129, 3072]
LW_M = [1, 63, 64, 65, 511, 512, 513, 1025, 8192]


def lora_wgrad_sweep(r):
    from qflux_b200 import lib
    c = Checks()
    for kd, Dp in enumerate(LW_DP):
        for km, M in enumerate(LW_M):
            seed = 1000 * kd + 10 * km + r
            tag = f"lora_wgrad r{r} Dp{Dp} M{M}"
            P = _mk(M, Dp + 3, seed=seed)[:, :Dp]                        # ldp = Dp + 3
            Qb = torch.full((M, 192), BIG, device="cuda", dtype=BF)
            Qb[:, 64:64 + r] = _mk(M, r, seed=seed + 1)
            Q = Qb[:, 64:64 + r]                                          # a column slice with ldq = 192, as the model's U slice
            ref, mag = lora_wgrad_ref(P, Q, r)
            inits = [_init(Dp * r, seed + 2), _init(Dp * r, seed + 3)]
            strides = [(r, 1), (1, Dp)]                                  # dB [Dp, r] and the transposed dA [r, Dp] store

            def outputs():
                s = Slots([Dp * r, Dp * r])
                s[0].copy_(inits[0])
                s[1].copy_(inits[1])
                return s

            def check(var, s):
                for k, (gi, gj) in enumerate(strides):
                    i0 = torch.as_strided(inits[k], (Dp, r), (gi, gj)).double()
                    _bound(c, f"lora_wgrad_{var}_max_err_over_bound", f"{tag} {var} store {k}", torch.as_strided(s[k], (Dp, r), (gi, gj)),
                           i0 + ref, RED_TOL * (i0.abs() + mag))
                _sentinels(c, f"{tag} {var}", s.buf, s.free, SENT)

            def atomic(s):
                for k, (gi, gj) in enumerate(strides):
                    lib.lora_wgrad(P, Q, s[k], gi, gj, r)

            def det(s, scr):
                for k, (gi, gj) in enumerate(strides):
                    lib.lora_wgrad_det(P, Q, s[k], gi, gj, r, scratch=scr)
            _run_both(c, tag, atomic, det, lib.det_scratch_wgrad(M, Dp, r), outputs, check)
    return c.out()


# ============================================================================ qfx_mod_grad
FORMS = ("sum", "sum_prod_stats", "prod_m")  # d shift; d shift + d scale (m = LN input, row statistics); d gate (m = branch output)


def _mod_grad_one(c, B, rpb, D, form, seed):
    from qflux_b200 import lib
    tag = f"mod_grad B{B} rpb{rpb} D{D} {form}"
    M = B * rpb
    g = _mk(M, D + 16, seed=seed)[:, 8:8 + D]                              # ldg = D + 16, base 16 bytes into the row
    m = mean = rstd = None
    if form != "sum":
        m = _mk(M, D + 24, seed=seed + 1, scale=2.0, shift=0.5)[:, :D]       # ldm = D + 24
    if form == "sum_prod_stats":
        mf = m.float()
        mean, rstd = mf.mean(1).contiguous(), torch.rsqrt(mf.var(1, unbiased=False) + 1e-6).contiguous()
    ref = mod_grad_ref(g, rpb, m, mean, rstd)
    chunks = {"sum": [(0, "sum")], "sum_prod_stats": [(0, "sum"), (1, "prod")], "prod_m": [(2, "prod")]}[form]
    inits = {k: _init(B * D, seed + 5 + k).view(B, D) for k, _ in chunks}

    def outputs():
        s = Slots([B * 6 * D])                                              # [B, 6D] (ldo = 6D): the other chunks keep SENT
        o, free = s[0].view(B, 6 * D), s.free[s.offs[0]:s.offs[0] + B * 6 * D].view(B, 6 * D)
        free[:] = True
        for k, _ in chunks:
            o[:, k * D:(k + 1) * D] = inits[k]
            free[:, k * D:(k + 1) * D] = False
        return s

    def check(var, s):
        o = s[0].view(B, 6 * D)
        for k, what in chunks:
            i0 = inits[k].double()
            b = RED_TOL * (i0.abs() + ref[what + "_mag"]) + (ref["flip"] if what == "prod" else 0)
            _bound(c, f"mod_grad_{var}_max_err_over_bound", f"{tag} {var} {what}", o[:, k * D:(k + 1) * D], i0 + ref[what], b)
        _sentinels(c, f"{tag} {var}", s.buf, s.free, SENT)

    def kw(s):
        o = s[0].view(B, 6 * D)
        pick = {what: o[:, k * D:(k + 1) * D] for k, what in chunks}
        return dict(sum_out=pick.get("sum"), m=m, prod_out=pick.get("prod"), mean=mean, rstd=rstd)
    _run_both(c, tag, lambda s: lib.mod_grad(g, rpb, **kw(s)), lambda s, scr: lib.mod_grad_det(g, rpb, **kw(s), scratch=scr),
              lib.det_scratch_mod_grad(M, rpb, D), outputs, check)


def mod_grad_sweep(D):
    c = Checks()
    sms = num_sms()
    c.res["sms"], c.res["plans"] = sms, []
    k = 0
    for B in (1, 3, 8):
        for rpb in (1, 31, 32, 33, 352, 1025):
            c.res["plans"].append(dict(mod_grad_plan(rpb, B, D, sms), B=B))
            for form in FORMS:
                _mod_grad_one(c, B, rpb, D, form, seed=17 * k + 3)
                k += 1
    return c.out()


def mod_grad_edges(B, D):
    c = Checks()
    sms = num_sms()
    edges = split_edges(lambda v: mod_grad_plan(v, B, D, sms), 33, 1 << 15, 8)  # the unit: one row for each of the CTA's 8 warps
    c.res["sms"], c.res["edges"], c.res["plans"] = sms, edges, {}
    S = _cdiv(4 * sms, _cdiv(D, 256) * B)
    want = {"mult64", "fill_minus1", "fill_plus1"} | ({"last_one_row"} if S >= 33 else set()) | ({"last_one_kblock"} if S >= 26 else set())
    c.res["unreachable"] = sorted({"last_one_row", "last_one_kblock"} - want)
    c.check(want <= set(edges), f"split edges not all found: {sorted(edges)} of {sorted(want)}")
    for k, (name, rpb) in enumerate(sorted(edges.items())):
        c.res["plans"][name] = mod_grad_plan(rpb, B, D, sms)
        for j, form in enumerate(FORMS):
            _mod_grad_one(c, B, rpb, D, form, seed=500 + 7 * k + j)
    return c.out()


# ============================================================================ qfx_flow_loss
def flow_loss_sweep(B, L):
    from qflux_b200 import lib
    c = Checks()
    k = 0
    for Ltot in sorted({L, L + 3, 2 * L}):
        for C in (16, 64):
            x0, noise = _mk(B, L, C, seed=k + 1), _mk(B, L, C, seed=k + 2)
            pred = _mk(B, Ltot, C, seed=k + 3)
            wt = torch.rand(B, L, device="cuda", generator=torch.Generator(device="cuda").manual_seed(k)) + 0.5
            norm = 1.0 / (B * L * C)
            for use_w in (False, True):
                for gs in (1.0, 0.25):
                    for with_dpred in (False, True):
                        k += 1
                        tag = f"flow_loss B{B} L{L} Ltot{Ltot} C{C} w{int(use_w)} gs{gs} dpred{int(with_dpred)}"
                        w = wt if use_w else None
                        loss64, lmag, rule, dp64 = flow_loss_ref(pred, x0, noise, w, norm, gs)
                        n = B * Ltot * C
                        outs = {}
                        for var in ("atomic", "det", "det_repeat"):
                            lbuf = torch.full((2 * GAP + 1,), SENT, device="cuda")
                            lbuf[GAP] = 1e30
                            dbuf = torch.full((n + 2 * GAP,), SENT_BF, device="cuda", dtype=BF)
                            dbuf[GAP:GAP + n] = 3.0
                            loss, dpred = lbuf[GAP:GAP + 1], (dbuf[GAP:GAP + n].view(B, Ltot, C) if with_dpred else None)
                            if var == "atomic":
                                lib.flow_loss(pred, x0, noise, w, norm, loss, dpred, gs)
                            else:
                                scr = torch.full((lib.DET_LOSS_PARTIALS,), float("nan"), device="cuda")
                                lib.flow_loss_det(pred, x0, noise, w, norm, loss, dpred, gs, scratch=scr)
                            outs[var] = (lbuf, dbuf)
                        torch.cuda.synchronize()
                        for var in ("atomic", "det"):
                            lbuf, dbuf = outs[var]
                            _bound(c, f"flow_loss_{var}_max_err_over_bound", f"{tag} {var} loss", lbuf[GAP:GAP + 1], loss64.reshape(1),
                                   (RED_TOL * lmag).reshape(1))
                            keep = torch.ones(2 * GAP + 1, dtype=torch.bool, device="cuda")
                            keep[GAP] = False
                            _sentinels(c, f"{tag} {var} loss", lbuf, keep, SENT)
                            dv = dbuf[GAP:GAP + n].view(B, Ltot, C)
                            if with_dpred:
                                same = _bits(dv[:, :L]) == _bits(rule[:, :L])
                                c.check(bool(same.all()), f"{tag} {var}: dpred differs from the fp32 rule at {int((~same).sum())} elements")
                                c.check(bool((_bits(dv[:, L:]) == 0).all()), f"{tag} {var}: dpred rows t >= L are not +0")
                                _bound(c, f"flow_dpred_{var}_max_err_over_ulp", f"{tag} {var} dpred vs fp64", dv[:, :L], dp64[:, :L],
                                       _up(dp64[:, :L]))
                            else:
                                c.check(bool((dv == 3.0).all()), f"{tag} {var}: dpred written although absent")
                            keep = torch.ones(n + 2 * GAP, dtype=torch.bool, device="cuda")
                            keep[GAP:GAP + n] = False
                            _sentinels(c, f"{tag} {var} dpred", dbuf, keep, SENT_BF)
                        c.check(torch.equal(_bits(outs["det"][0]), _bits(outs["det_repeat"][0])) and
                                torch.equal(_bits(outs["det"][1]), _bits(outs["det_repeat"][1])), f"{tag}: det twin differs between launches")
    c.res["combinations"] = k
    return c.out()


# ============================================================================ qfx_gemv_act
GV_N = [1, 2, 3, 5, 64, 3072, 147459]  # 147459: every warp of the persistent grid loops several times; the tail is not a multiple of 4


def gemv_kmax(B):
    """the largest K (multiple of 8) whose fp32 staging of act(x), B * K * 4 bytes, fits the kernel's 200 KiB"""
    return 200 * 1024 // (4 * B) // 8 * 8


def gemv_sweep(B):
    from qflux_b200 import lib
    c = Checks()
    Ks = [8, 256, 768, 3072, gemv_kmax(B)]
    c.res["K"], c.res["skipped"] = Ks, []
    k = 0
    for N in GV_N:
        for K in Ks:
            if N * K > 1_000_000_000:  # an fp64 copy of W would need more than 8 GB
                c.res["skipped"].append([N, K])
                continue
            k += 1
            x = _mk(B, K + 8, seed=k, scale=2.0)[:, :K]                      # ldx = K + 8
            W = _mk(N, K, seed=k + 1, scale=K ** -0.5)
            bias_t = _mk(N, seed=k + 2)
            for act in (0, 1):
                for use_bias in (False, True):
                    tag = f"gemv_act B{B} N{N} K{K} act{act} bias{int(use_bias)}"
                    bias = bias_t if use_bias else None
                    ldy = N + 3
                    buf = torch.full((B * ldy + 2 * GAP,), SENT_BF, device="cuda", dtype=BF)
                    y = buf[GAP:GAP + B * ldy].view(B, ldy)[:, :N]              # a slice with ldy > N: sentinels past N in each row
                    lib.gemv_act(x, W, bias, y, act)
                    ref, mag, flip = gemv_ref(x, W, bias, act)
                    big = torch.maximum(y.double().abs(), ref.abs())
                    _bound(c, "gemv_act_max_err_over_bound", tag, y, ref, RED_TOL * mag + flip + _up(big))
                    keep = torch.ones(B * ldy + 2 * GAP, dtype=torch.bool, device="cuda")
                    keep[GAP:GAP + B * ldy].view(B, ldy)[:, :N] = False
                    _sentinels(c, tag, buf, keep, SENT_BF)
                    del ref, mag, flip
    c.res["shapes"] = k
    return c.out()


CASES = {}
for _G in (1, 2, 3):
    CASES[f"wgrad_tc_mode0_G{_G}"] = (lambda G: lambda: wgrad_tc_sweep(0, G))(_G)
for _G in (2, 3):
    for _Dg in (128, 3072):
        CASES[f"wgrad_tc_mode1_G{_G}_Dg{_Dg}"] = (lambda G, Dg: lambda: wgrad_tc_sweep(1, G, Dg))(_G, _Dg)
for _Na in (128, 3072):
    CASES[f"wgrad_tc_edges_Na{_Na}"] = (lambda Na: lambda: wgrad_tc_edges(Na))(_Na)
for _r in (4, 8, 16, 32, 64):
    CASES[f"lora_wgrad_r{_r}"] = (lambda r: lambda: lora_wgrad_sweep(r))(_r)
for _D in (8, 264, 3072):
    CASES[f"mod_grad_D{_D}"] = (lambda D: lambda: mod_grad_sweep(D))(_D)
for _B, _D in ((1, 3072), (3, 264), (8, 3072)):
    CASES[f"mod_grad_edges_B{_B}_D{_D}"] = (lambda B, D: lambda: mod_grad_edges(B, D))(_B, _D)
for _B in (1, 4):
    for _L in (1, 7, 1024, 4096):
        CASES[f"flow_loss_B{_B}_L{_L}"] = (lambda B, L: lambda: flow_loss_sweep(B, L))(_B, _L)
for _B in range(1, 9):
    CASES[f"gemv_act_B{_B}"] = (lambda B: lambda: gemv_sweep(B))(_B)

if __name__ == "__main__":
    main(CASES, os.path.abspath(__file__), "reduce_check.log")
