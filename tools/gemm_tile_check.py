"""GPU check of qfx_gemm_bf16 per output tile and per row, against

  (a) an fp64 reference of the same contraction and epilogue (from the kernel's bf16 inputs), next to the same operation in bf16
      eager on the device (torch bf16 matmul, then the epilogue with eager bf16 rounding), which sets the scale of "close":
      err_kernel <= C * err_eager + FLOOR (relative L2 against fp64) in every (problem, 128-row m-tile, block_n n-tile) and in
      every output row;
  (b) the epilogue's stated rounding rule applied to the kernel's own accumulator, read back through EPI_BIAS on the same inputs
      (same problems, same block_n, so the same k order).  The read-back returns the kernel's first rounding point exactly:
      bf16(acc + bias) for GELU / RESID_GATE, bf16(alpha * acc) for ADD / DGELU / ATTN_DO.  Everything after it is elementwise:
      data movement (out2 copies, the ATTN_DO head-major scatter) and the fp32 add / multiply chains of RESID_GATE and ADD must
      match the rule bit for bit, the GELU / GELU' epilogues (tanhf) within one ulp of the output, and delta within RED_TOL of
      the sum of its terms.  A moved rounding point fails here at once, far below what an L2 norm can see;
  (c) sentinels: outputs are filled with a NaN pattern first; columns outside a problem's slice, rows past M, joint positions of
      dO_joint / delta that no row group covers must keep it, dead rows of ragged bands must be exact zeros;
  (d) tests/emu_lib.py on CPU copies of the inputs: sentinels and dead rows bit-identical, values within the rounding-flip bound
      (the emulation sums in another order, so a rounded intermediate may land on the neighbouring bf16 value).

Each case returns a dict of measurements plus `fail`, the list of violated checks (each names its problem, tile or row).  Run
stand-alone: `python tools/gemm_tile_check.py [case ...]` (one subprocess per case).

Every launch here has fewer tiles than an H100 has SMs, so each CTA of the persistent kernel computes exactly one tile.  What
happens between a CTA's tiles (the ring carried over, the next tile's problem and k-block count, the epilogue overlapped with the
next tile's loads) is checked by tools/gemm_sched_check.py, which runs `run` on launches with several tiles per CTA.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from harness import ROOT, main  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from glue_check import RED_TOL, Checks, _mk, _up  # noqa: E402

BF, F64 = torch.bfloat16, torch.float64
EPI_BIAS, EPI_GELU, EPI_RESID_GATE, EPI_DGELU, EPI_ADD, EPI_ATTN_DO = 0, 1, 2, 3, 4, 5
EPI_NAME = {0: "bias", 1: "gelu", 2: "resid_gate", 3: "dgelu", 4: "add", 5: "attn_do"}
# err_kernel <= C * err_eager + FLOOR, relative L2 against fp64, per tile and per row (ratios measured on an H100: see the commit
# message that introduced this file)
C_TILE, FLOOR_TILE = 1.5, 1e-4
C_ROW, FLOOR_ROW = 1.75, 5e-4
SENT_BITS = 0x7FC1  # a quiet NaN no kernel produces: a sentinel that survives a launch proves the position was not written
SENT_F32 = -7.25
PADC = 64           # sentinel columns on each side of a problem's output slice
PADR = 3            # sentinel rows past M
DEV = "cuda"


def sentinel(*shape, device=None):
    device = device or DEV
    return torch.full(shape, SENT_BITS, dtype=torch.int16, device=device).view(BF)


def is_sent(t):
    return t.contiguous().view(torch.int16) == SENT_BITS


def same(a, b):
    """element-wise equality of values (-0 == +0); NaN only equals NaN"""
    a, b = a.float(), b.float()
    return (a == b) | (a.isnan() & b.isnan())


def row_rel_max(a, ref):
    """worst per-row relative L2 of 2-D a against ref"""
    a, ref = a.double(), ref.double()
    return ((a - ref).norm(dim=1) / ref.norm(dim=1).clamp_min(1e-300)).max().item()


# ============================================================================ fp64 references (device-agnostic; checked on CPU too)
def gelu64(u):
    return 0.5 * u * (1 + torch.tanh(0.7978845608028654 * (u + 0.044715 * u ** 3)))


def gelu_grad64(u):
    k0, k1 = 0.7978845608028654, 0.044715
    t = torch.tanh(k0 * (u + k1 * u ** 3))
    return 0.5 * (1 + t) + 0.5 * u * (1 - t * t) * k0 * (1 + 3 * k1 * u * u)


def acc_ref(p, N, trans_b, lora_group_n=0, dt=F64):
    """A.B(^T) + the LoRA k-blocks (A2 columns a2_col0 + (g*kb2 + j)*64 for output group g), in dtype dt"""
    A, W = p["A"].to(dt), p["B"].to(dt)
    acc = A @ (W if trans_b else W.t())
    kb2 = p.get("kb2", 0)
    if kb2:
        w2, c0 = 64 * kb2, p.get("a2_col0", 0)
        A2, B2 = p["A2"].to(dt), p["B2"].to(dt)
        if trans_b:
            acc = acc + A2[:, c0:c0 + w2] @ B2[:w2]
        else:
            groups = N // lora_group_n if lora_group_n else 1
            gn = N // groups
            for g in range(groups):
                acc[:, g * gn:(g + 1) * gn] += A2[:, c0 + g * w2:c0 + (g + 1) * w2] @ B2[g * gn:(g + 1) * gn, :w2].t()
    return acc


def gate_rows(p, M):
    return p["gate"].repeat_interleave(p.get("rows_per_batch") or M, 0)[:M]


def epi_ref(p, acc, epi, alpha):
    """fp64 epilogue: {"out": [M, N], "out2": [M, N] or absent}; for ATTN_DO "out" is g token-major (the scatter is data movement)"""
    M, dt = acc.shape[0], acc.dtype
    b = p["bias"].to(dt) if p.get("bias") is not None else 0.0
    if epi == EPI_BIAS:
        return dict(out=alpha * acc + b)
    if epi == EPI_GELU:
        u = acc + b
        return dict(out=gelu64(u), out2=u)
    if epi == EPI_RESID_GATE:
        y = acc + b
        return dict(out=p["resid"].to(dt) + gate_rows(p, M).to(dt) * y, out2=y)
    if epi == EPI_DGELU:
        return dict(out=alpha * acc * gelu_grad64(p["aux"].to(dt)))
    if epi == EPI_ADD:
        return dict(out=p["resid"].to(dt) + alpha * acc)
    if epi == EPI_ATTN_DO:
        g = alpha * acc
        return dict(out=g, out2=g, delta=(g * p["aux"].to(dt)).view(M, -1, 128).sum(-1))
    raise ValueError(epi)


def epi_eager(p, epi, alpha, trans_b, N, lora_group_n=0):
    """the same operation in bf16 eager: torch bf16 matmuls (+ the LoRA term as a second bf16 matmul), then the epilogue one bf16
    op at a time, as the reference's modules round"""
    A, W = p["A"], p["B"]
    acc = A @ (W if trans_b else W.t())
    kb2 = p.get("kb2", 0)
    if kb2:
        w2, c0 = 64 * kb2, p.get("a2_col0", 0)
        if trans_b:
            acc = acc + p["A2"][:, c0:c0 + w2] @ p["B2"][:w2]
        else:
            groups = N // lora_group_n if lora_group_n else 1
            gn = N // groups
            acc = torch.cat([acc[:, g * gn:(g + 1) * gn] + p["A2"][:, c0 + g * w2:c0 + (g + 1) * w2] @ p["B2"][g * gn:(g + 1) * gn, :w2].t()
                             for g in range(groups)], 1)
    M = acc.shape[0]
    sc = (lambda t: t * alpha) if alpha != 1.0 else (lambda t: t)
    b = p.get("bias")
    lin = acc + b if b is not None else acc
    if epi == EPI_BIAS:
        return dict(out=sc(acc) + b if b is not None else sc(acc))
    if epi == EPI_GELU:
        return dict(out=F.gelu(lin, approximate="tanh"), out2=lin)
    if epi == EPI_RESID_GATE:
        return dict(out=p["resid"] + gate_rows(p, M) * lin, out2=lin)
    if epi == EPI_DGELU:
        return dict(out=torch.ops.aten.gelu_backward(sc(acc), p["aux"], approximate="tanh"))
    if epi == EPI_ADD:
        return dict(out=p["resid"] + sc(acc))
    if epi == EPI_ATTN_DO:
        return dict(out=sc(acc), out2=sc(acc))
    raise ValueError(epi)


def rule(p, rb, epi):
    """the kernel's stated rounding rule applied to its own first rounding point rb (bf16, read back through EPI_BIAS):
    bit-exact expectation for out / out2 (GELU / DGELU: before their last rounding, in fp64)"""
    M = rb.shape[0]
    y = rb.float()
    if epi == EPI_GELU:
        return dict(out=gelu64(rb.double()), out2=rb)
    if epi == EPI_RESID_GATE:
        z = (gate_rows(p, M).float() * y).to(BF).float()
        return dict(out=(p["resid"].float() + z).to(BF), out2=rb)
    if epi == EPI_DGELU:
        return dict(out=rb.double() * gelu_grad64(p["aux"].double()))
    if epi == EPI_ADD:
        return dict(out=(p["resid"].float() + y).to(BF))
    if epi == EPI_ATTN_DO:
        return dict(out=rb, out2=rb)
    raise ValueError(epi)


# ============================================================================ one launch, every check
def _tile_of(M, bands, device):
    """the kernel's m-tile of every row (dense: row // 128; ragged: two tiles per 256-row band), and the live-row mask"""
    if bands is None:
        return torch.arange(M, device=device) // 128, None
    t = torch.zeros(M, dtype=torch.long, device=device)
    live = torch.zeros(M, dtype=torch.bool, device=device)
    for i, s in enumerate(bands.host_tiles):
        e = min(s + 256, M)
        t[s:e] = 2 * i + (torch.arange(s, e, device=device) - s) // 128
        live[s:e] = True
    return t, live


def _regions(c, name, k, e, ref, tile_of, bn, live=None, rows=True):
    """relative L2 of kernel and bf16 eager against fp64 per (m-tile, n-tile) and per row: err_k <= C * err_e + FLOOR (per row only
    when `rows`; the ratio is reported either way)"""
    if live is not None:
        k, e, ref, tile_of = k[live], e[live], ref[live], tile_of[live]
    ref = ref.double()
    dk, de, rr = (k.double() - ref) ** 2, (e.double() - ref) ** 2, ref ** 2
    M, N = ref.shape
    nt = N // bn

    def per_tile(x):
        s = x.view(M, nt, bn).sum(2)
        return torch.zeros(int(tile_of.max()) + 1, nt, dtype=F64, device=x.device).index_add_(0, tile_of, s)
    trr = per_tile(rr)
    used = trr > 0
    tk, te = (per_tile(dk) / trr.clamp_min(1e-300)).sqrt(), (per_tile(de) / trr.clamp_min(1e-300)).sqrt()
    rrr = rr.sum(1).clamp_min(1e-300)
    rk, re_ = (dk.sum(1) / rrr).sqrt(), (de.sum(1) / rrr).sqrt()
    c.res[f"{name}_tile_worst_k_e"] = [tk[used].max().item(), te[used].max().item()]
    c.res[f"{name}_tile_ratio_max"] = (tk / te.clamp_min(1e-300))[used].max().item()
    c.res[f"{name}_row_ratio_max"] = (rk / re_.clamp_min(1e-300)).max().item()
    bad = ~(tk <= C_TILE * te + FLOOR_TILE) & used
    for mt, n_t in bad.nonzero().tolist()[:3]:
        c.fail.append(f"{name} tile (m{mt}, n{n_t}): kernel {tk[mt, n_t].item():.3e} vs bf16 eager {te[mt, n_t].item():.3e}")
    row_id = torch.arange(M, device=ref.device) if live is None else live.nonzero().flatten()
    for i in (~(rk <= C_ROW * re_ + FLOOR_ROW)).nonzero().flatten().tolist()[:3] if rows else []:
        c.fail.append(f"{name} row {int(row_id[i])}: kernel {rk[i].item():.3e} vs bf16 eager {re_[i].item():.3e}")


def _exact(c, name, k, want):
    ok = same(k, want)
    c.res[f"{name}_bitfrac"] = ok.double().mean().item() if ok.numel() else 1.0
    if not bool(ok.all()):
        r = ok.view(ok.shape[0], -1).all(1).logical_not().nonzero().flatten()
        c.fail.append(f"{name}: {int((~ok).sum())} of {ok.numel()} elements differ from the rule, first rows {r[:4].tolist()}")


def gelu_fp32_err(epi, first, aux=None):
    """absolute error of evaluating GELU (on u = first) or g * GELU'(aux) (g = first) in fp32: 1 + tanh and 1 - tanh^2 cancel, and
    GELU' scales the tanh error by |x|^3"""
    if epi == EPI_GELU:
        return 2.0 ** -20 * (1 + first.abs())
    return 2.0 ** -20 * (1 + aux.abs()) ** 3 * first.abs()


def _ulp_bound(c, name, k, want64, fp32_err):
    """bf16 k within one ulp of the fp64 value the rule gives before its last rounding, plus fp32_err, the absolute error of
    evaluating the rule in fp32 (GELU and GELU' lose relative accuracy where 1 + tanh cancels)"""
    d = (k.double() - want64).abs()
    ok = d <= _up(torch.maximum(k.double().abs(), want64.abs())) + fp32_err
    c.res[f"{name}_rule_bitfrac"] = (k == want64.to(BF)).double().mean().item()
    if not bool(ok.all()):
        r = (~ok).any(1).nonzero().flatten()
        c.fail.append(f"{name}: {int((~ok).sum())} elements beyond one ulp of the rule, first rows {r[:4].tolist()}")


def run(c, tag, probs, N, K, *, trans_b, epi, alpha=1.0, bn, lora_group_n=0, attn=None, emu_check=True, alias=False, rows=True):
    """probs: list of dicts of device tensors (A, B, optional A2/B2/kb2/a2_col0, bias, resid, gate/rows_per_batch, aux, with_out2,
    bands, s_offset).  attn (ATTN_DO): dict(B, H, S).  alias (ADD): out is the resid buffer itself.  rows: hold every row to the
    per-row bound (see gemm_sched_check.py for launches whose rows are too short for it)."""
    from qflux_b200 import lib
    dev = probs[0]["A"].device
    full, lp = [], []
    if epi == EPI_ATTN_DO:
        dOj = sentinel(attn["B"], attn["H"], attn["S"], 128)
        delta = torch.full((attn["B"], attn["H"], attn["S"]), SENT_F32, device=dev)
    for p in probs:
        M = p["A"].shape[0]
        if alias:
            f = sentinel(M + PADR, N + 2 * PADC)
            f[:M, PADC:PADC + N] = p["resid"]
            p["resid_in"] = p["resid"].clone()
            p["resid"] = f[:M, PADC:PADC + N]
        else:
            f = sentinel(M + PADR, N + 2 * PADC)
        f2 = sentinel(M + PADR, N + 2 * PADC) if (epi == EPI_GELU or p.get("with_out2")) else None
        full.append((f, f2))
        out = dOj if epi == EPI_ATTN_DO else f[:M, PADC:PADC + N]
        lp.append(lib.gemm_problem(p["A"], p["B"], out, A2=p.get("A2"), B2=p.get("B2"), kb2=p.get("kb2", 0), a2_col0=p.get("a2_col0", 0),
                                   bias=p.get("bias"), out2=None if f2 is None else f2[:M, PADC:PADC + N], resid=p.get("resid"),
                                   gate=p.get("gate"), rows_per_batch=p.get("rows_per_batch", 0), aux=p.get("aux"),
                                   row_bands=p.get("bands"), delta=delta if epi == EPI_ATTN_DO else None, s_offset=p.get("s_offset", 0)))
    lib.gemm(lp, N, K, trans_b=trans_b, epilogue=epi, alpha=alpha, lora_group_n=lora_group_n, block_n=bn)
    # the kernel's own first rounding point, through EPI_BIAS on the same problems and block_n
    rbs, lr = [], []
    rb_alpha = 1.0 if epi in (EPI_GELU, EPI_RESID_GATE) else alpha
    for p in probs:
        rb = sentinel(p["A"].shape[0], N)
        rbs.append(rb)
        lr.append(lib.gemm_problem(p["A"], p["B"], rb, A2=p.get("A2"), B2=p.get("B2"), kb2=p.get("kb2", 0), a2_col0=p.get("a2_col0", 0),
                                   bias=p.get("bias") if epi in (EPI_GELU, EPI_RESID_GATE) else None, row_bands=p.get("bands")))
    if epi != EPI_BIAS:
        lib.gemm(lr, N, K, trans_b=trans_b, epilogue=EPI_BIAS, alpha=rb_alpha, lora_group_n=lora_group_n, block_n=bn)
    if dev.type == "cuda":
        torch.cuda.synchronize()
    covered = torch.zeros(attn["S"], dtype=torch.bool, device=dev) if epi == EPI_ATTN_DO else None
    results = []
    for i, p in enumerate(probs):
        M = p["A"].shape[0]
        f, f2 = full[i]
        if epi == EPI_ATTN_DO:
            rpb, so = p["rows_per_batch"], p["s_offset"]
            nb = M // rpb
            got = dict(out=dOj[:nb, :, so:so + rpb].permute(0, 2, 1, 3).reshape(M, N),
                       delta=delta[:nb, :, so:so + rpb].permute(0, 2, 1).reshape(M, -1))
            covered[so:so + rpb] = True
        else:
            got = dict(out=f[:M, PADC:PADC + N])
        if f2 is not None:
            got["out2"] = f2[:M, PADC:PADC + N]
        if epi == EPI_BIAS:
            rbs[i] = got["out"]
        results.append(got)
        pr = dict(p, resid=p.get("resid_in", p.get("resid")))
        tile_of, live = _tile_of(M, p.get("bands"), dev)
        ref = epi_ref(pr, acc_ref(pr, N, trans_b, lora_group_n), epi, alpha)
        eag = epi_eager(pr, epi, alpha, trans_b, N, lora_group_n)
        pn = f"{tag}_p{i}"
        for o in got:
            if o == "delta":
                continue
            _regions(c, f"{pn}_{o}", got[o], eag[o], ref[o], tile_of, bn, live, rows)
        # (b) the stated rounding rule on the kernel's own accumulator
        if epi != EPI_BIAS:
            want = rule(pr, rbs[i], epi)
            sel = (lambda t: t) if live is None else (lambda t: t[live])
            for o in got:
                if o == "delta":
                    g = rbs[i].double().view(M, -1, 128)
                    aux = p["aux"].double().view(M, -1, 128)
                    d = (got["delta"].double() - (g * aux).sum(-1)).abs()
                    mag = (g * aux).abs().sum(-1)
                    c.res[f"{pn}_delta_max_rel"] = (d / mag.clamp_min(1e-30)).max().item()
                    c.check(bool((d <= RED_TOL * mag + 1e-30).all()), f"{pn}_delta: beyond {RED_TOL} of sum |g * O| against the rule")
                elif want[o].dtype == F64:
                    err = gelu_fp32_err(epi, rbs[i].double(), p["aux"].double() if epi == EPI_DGELU else None)
                    _ulp_bound(c, f"{pn}_{o}", sel(got[o]), sel(want[o]), sel(err))
                else:
                    _exact(c, f"{pn}_{o}", sel(got[o]), sel(want[o]))
        # (c) sentinels and dead rows
        for o, buf in (("out", f), ("out2", f2)):
            if buf is None or (o == "out" and epi == EPI_ATTN_DO):
                continue
            inner = torch.zeros_like(buf, dtype=torch.bool)
            inner[:M, PADC:PADC + N] = True
            c.check(bool(is_sent(buf)[~inner].all()), f"{pn}_{o}: written outside its rows / column slice")
            if live is not None:
                c.check(bool((buf[:M, PADC:PADC + N][~live] == 0).all()), f"{pn}_{o}: dead rows of the ragged bands are not exact zeros")
    if epi == EPI_ATTN_DO:
        c.check(bool(is_sent(dOj[:, :, ~covered]).all()), f"{tag}: dO_joint written at joint positions no row group covers")
        c.check(bool((delta[:, :, ~covered] == SENT_F32).all()), f"{tag}: delta written at joint positions no row group covers")
        c.res[f"{tag}_uncovered_positions"] = int((~covered).sum())
    if emu_check:
        _vs_emu(c, tag, probs, full, N, K, trans_b, epi, alpha, lora_group_n, attn, dOj if epi == EPI_ATTN_DO else None,
                delta if epi == EPI_ATTN_DO else None, alias)
    return results


def _vs_emu(c, tag, probs, full, N, K, trans_b, epi, alpha, lora_group_n, attn, dOj, delta, alias):
    """tests/emu_lib.py on CPU copies: positions the kernel must not write (sentinels, zero-filled dead rows) bit-identical,
    values within the rounding-flip bound of the emulation's intermediates"""
    from qflux_b200 import lib
    import emu_lib as emu
    cpu = lambda t: None if t is None else t.cpu()
    efull, ep = [], []
    if epi == EPI_ATTN_DO:
        edOj = sentinel(attn["B"], attn["H"], attn["S"], 128, device="cpu")
        edelta = torch.full((attn["B"], attn["H"], attn["S"]), SENT_F32)
    for p, (f, f2) in zip(probs, full):
        M = p["A"].shape[0]
        ef = sentinel(M + PADR, N + 2 * PADC, device="cpu")
        if alias:
            ef[:M, PADC:PADC + N] = p["resid_in"].cpu()
        ef2 = None if f2 is None else sentinel(M + PADR, N + 2 * PADC, device="cpu")
        efull.append((ef, ef2))
        bands = p.get("bands")
        ep.append(emu.gemm_problem(cpu(p["A"]), cpu(p["B"]), edOj if epi == EPI_ATTN_DO else ef[:M, PADC:PADC + N], A2=cpu(p.get("A2")),
                                   B2=cpu(p.get("B2")), kb2=p.get("kb2", 0), a2_col0=p.get("a2_col0", 0), bias=cpu(p.get("bias")),
                                   out2=None if ef2 is None else ef2[:M, PADC:PADC + N],
                                   resid=ef[:M, PADC:PADC + N] if alias else cpu(p.get("resid")), gate=cpu(p.get("gate")),
                                   rows_per_batch=p.get("rows_per_batch", 0), aux=cpu(p.get("aux")),
                                   row_bands=bands, delta=edelta if epi == EPI_ATTN_DO else None, s_offset=p.get("s_offset", 0)))
    emu.gemm(ep, N, K, trans_b=trans_b, epilogue=epi, alpha=alpha, lora_group_n=lora_group_n)
    flips = []
    for i, p in enumerate(probs):
        M = p["A"].shape[0]
        pr = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in dict(p, resid=p.get("resid_in", p.get("resid"))).items()}
        acc = acc_ref(pr, N, trans_b, lora_group_n, torch.float32)  # the emulation's accumulator (fp32, CPU)
        absp = {k: (v.abs() if torch.is_tensor(v) and k in ("A", "B", "A2", "B2") else v) for k, v in pr.items()}
        pre = RED_TOL * acc_ref(absp, N, trans_b, lora_group_n, F64) * abs(alpha)  # fp32 reduction-order allowance
        b = pr["bias"].double() if pr.get("bias") is not None else 0.0
        first = (acc.double() * (alpha if epi not in (EPI_GELU, EPI_RESID_GATE) else 1.0) + (b if epi in (EPI_BIAS, EPI_GELU, EPI_RESID_GATE) else 0.0))
        d1 = pre + _up(first)  # the first rounding point may flip
        (ef, ef2), (f, f2) = efull[i], full[i]
        if epi == EPI_ATTN_DO:
            rpb, so = p["rows_per_batch"], p["s_offset"]
            nb = M // rpb
            pick = lambda t: t[:nb, :, so:so + rpb].permute(0, 2, 1, 3).reshape(M, N)
            k_out, e_out = pick(dOj).cpu(), pick(edOj)
        else:
            k_out, e_out = f[:M, PADC:PADC + N].cpu(), ef[:M, PADC:PADC + N]
        big = torch.maximum(k_out.double().abs(), e_out.double().abs())
        if epi == EPI_BIAS:
            bd = d1 + _up(big)
        elif epi == EPI_GELU:
            bd = 1.2 * d1 + _up(big) + 2 * gelu_fp32_err(epi, first.abs() + d1)
        elif epi == EPI_RESID_GATE:
            g = gate_rows(pr, M).double().abs()
            bd = g * d1 + _up(g * first.abs()) + _up(big)
        elif epi == EPI_DGELU:
            bd = d1 * gelu_grad64(pr["aux"].double()).abs() + _up(big) + 2 * gelu_fp32_err(epi, first.abs() + d1, pr["aux"].double())
        elif epi == EPI_ADD:
            bd = d1 + _up(big)
        else:
            bd = d1
        outs = [("out", k_out, e_out, bd)]
        if f2 is not None:
            outs.append(("out2", f2[:M, PADC:PADC + N].cpu(), ef2[:M, PADC:PADC + N], d1))
        for o, k, e, bound in outs:
            d = (k.double() - e.double()).abs()
            live = p.get("bands")
            ok = d <= bound
            if live is not None:
                _, lv = _tile_of(M, live, "cpu")
                ok = torch.where(lv[:, None], ok, same(k, e))
            flips.append((d == 0).double().mean().item())
            c.res[f"emu_{tag}_p{i}_{o}_bitfrac"] = flips[-1]
            c.res[f"emu_{tag}_p{i}_{o}_max_over_bound"] = (d / bound).max().item()
            c.check(bool(ok.all()), f"emu_{tag}_p{i}_{o}: {int((~ok).sum())} elements beyond the rounding-flip bound")
        for o, kb, eb in (("out", f, ef), ("out2", f2, ef2)):
            if kb is None or (o == "out" and epi == EPI_ATTN_DO):
                continue
            inner = torch.zeros_like(eb, dtype=torch.bool)
            inner[:M, PADC:PADC + N] = True
            c.check(bool(same(kb.cpu()[~inner], eb[~inner]).all()), f"emu_{tag}_p{i}_{o}: outside positions differ from the kernel")
        if epi == EPI_ATTN_DO:
            g = e_out.double().view(M, -1, 128)
            aux = pr["aux"].double().view(M, -1, 128)
            kd = delta[:nb, :, so:so + rpb].permute(0, 2, 1).reshape(M, -1).cpu().double()
            ed = edelta[:nb, :, so:so + rpb].permute(0, 2, 1).reshape(M, -1).double()
            tol = RED_TOL * (g * aux).abs().sum(-1) + (aux.abs() * d1.view(M, -1, 128)).sum(-1)  # sum order + flips of g
            c.check(bool(((kd - ed).abs() <= tol).all()), f"emu_{tag}_p{i}_delta: beyond the reduction + flip bound")
    if epi == EPI_ATTN_DO:
        c.check(bool(is_sent(dOj).cpu().eq(is_sent(edOj)).all()), f"emu_{tag}: dO_joint coverage differs from the kernel")
        c.check(bool((delta.cpu() == SENT_F32).eq(edelta == SENT_F32).all()), f"emu_{tag}: delta coverage differs from the kernel")


# ============================================================================ operands
def _prob(M, N, K, trans_b, seed, *, kb2=0, a2_col0=0, groups=1, bias=False, epi=EPI_BIAS, rows_per_batch=0, with_out2=False,
          shift=0.0, device=None):
    """one problem's operands; `shift` moves this problem's epilogue operands away from the others' (a misrouted tile is off by O(1))"""
    device = device or DEV
    p = dict(A=_mk(M, K, seed=seed, device=device),
             B=_mk(K, N, seed=seed + 1, scale=K ** -0.5, device=device) if trans_b else _mk(N, K, seed=seed + 1, scale=K ** -0.5, device=device))
    if kb2:
        p.update(A2=_mk(M, a2_col0 + 64 * kb2 * groups + 64, seed=seed + 2, device=device), kb2=kb2, a2_col0=a2_col0,
                 B2=_mk(64 * kb2, N, seed=seed + 3, scale=0.125, device=device) if trans_b else _mk(N, 64 * kb2, seed=seed + 3, scale=0.125, device=device))
    if bias:
        p["bias"] = _mk(N, seed=seed + 4, shift=shift, device=device)
    if epi in (EPI_RESID_GATE, EPI_ADD):
        p["resid"] = _mk(M, N, seed=seed + 5, scale=2.0, shift=shift, device=device)
    if epi == EPI_RESID_GATE:
        rpb = rows_per_batch or M
        p["gate"] = _mk(-(-M // rpb), 3 * N, seed=seed + 6, scale=0.5, shift=1.0 + shift, device=device)[:, N:2 * N]
        p["rows_per_batch"] = rpb
    if epi in (EPI_DGELU, EPI_ATTN_DO):
        p["aux"] = _mk(M, N, seed=seed + 7, scale=1.5, shift=shift, device=device)
    if with_out2:
        p["with_out2"] = True
    return p


def epilogue_case(epi, trans_b, bn):
    """one epilogue at one block_n: four problems with M = 1, 127, 129, 300 (one with a LoRA k-block, one with out2 and a gate /
    batch boundary inside a tile), at K = 64 (one k-block) and K = 12288 (many turns of the TMA ring); alpha != 1 where it applies"""
    c = Checks()
    alpha = 1.0 if epi in (EPI_GELU, EPI_RESID_GATE) else 0.75
    N = 2 * bn
    for K in (64, 12288):
        if epi == EPI_ATTN_DO:  # B = 3 samples; row groups at joint offsets 0, 43, 45 leave position 44 and a tail uncovered
            H, B = N // 128, 3
            spec = [(43, 0), (1, 43), (100, 45)]
            probs = [_prob(B * r, N, K, True, 10 * i + 1, epi=epi, kb2=1 if i == 2 else 0, with_out2=i == 2, shift=i) for i, (r, _) in enumerate(spec)]
            for p, (r, so) in zip(probs, spec):
                p.update(rows_per_batch=r, s_offset=so)
            run(c, f"K{K}", probs, N, K, trans_b=True, epi=epi, alpha=alpha, bn=bn, attn=dict(B=B, H=H, S=148))
            continue
        probs = []
        for i, M in enumerate((1, 127, 129, 300)):
            probs.append(_prob(M, N, K, trans_b, 10 * i + 1, epi=epi, bias=epi in (EPI_BIAS, EPI_GELU, EPI_RESID_GATE), kb2=1 if i == 2 else 0,
                               a2_col0=64 if i == 2 else 0, rows_per_batch=97 if M == 300 else 0, with_out2=(M == 300 and epi == EPI_RESID_GATE),
                               shift=0.5 * i))
        run(c, f"K{K}", probs, N, K, trans_b=trans_b, epi=epi, alpha=alpha, bn=bn)
    return c.out()


def add_alias_case():
    """FLUX single-block backward (flux_model.py): d xm = dgrad(qkv) + dgrad(proj_mlp) with EPI_ADD writing into its own resid,
    N = D, K = 4D at a reduced D; and the same launch not aliased"""
    c = Checks()
    D, M = 384, 600
    for bn in (128, 192):
        for alias in (True, False):
            probs = [_prob(M, D, 4 * D, True, 1, epi=EPI_ADD)]
            run(c, f"bn{bn}_{'alias' if alias else 'sep'}", probs, D, 4 * D, trans_b=True, epi=EPI_ADD, bn=bn, alias=alias)
    return c.out()


def lora_col0_case():
    """LoRA k-blocks taken from A2 columns a2_col0 + (g*kb2 + j)*64: three output groups (fused q|k|v) with kb2 = 1, 2, 3, and the
    trans_b dgrad with a2_col0 > 0.  A2 carries 64 extra columns on each side, so ignoring a2_col0 reads different data."""
    c = Checks()
    for kb2 in (1, 2, 3):
        probs = [_prob(300, 384, 256, False, 1, kb2=kb2, a2_col0=64, groups=3, bias=True), _prob(129, 384, 256, False, 11, kb2=kb2, a2_col0=128, groups=3)]
        run(c, f"nt_kb{kb2}", probs, 384, 256, trans_b=False, epi=EPI_BIAS, alpha=0.5, bn=128, lora_group_n=128)
        probs = [_prob(300, 256, 256, True, 1, kb2=kb2, a2_col0=64 * kb2)]
        run(c, f"nn_kb{kb2}", probs, 256, 256, trans_b=True, epi=EPI_BIAS, alpha=0.5, bn=128)
    return c.out()


def six_case(epi, trans_b):
    """six problems in one launch, M = 1 / 700 mixed, each with its own operands shifted apart: a tile routed to the wrong problem
    (tiles_m_end) is off by O(1) in that tile alone"""
    c = Checks()
    Ms = (1, 700, 129, 1, 300, 127)
    N, K = 256, 320
    probs = [_prob(M, N, K, trans_b, 10 * i + 1, epi=epi, bias=epi in (EPI_BIAS, EPI_GELU, EPI_RESID_GATE), shift=1.5 * i,
                   rows_per_batch=100 if M == 700 else 0) for i, M in enumerate(Ms)]
    run(c, "six", probs, N, K, trans_b=trans_b, epi=epi, alpha=1.0 if epi in (EPI_GELU, EPI_RESID_GATE) else 0.5, bn=128)
    return c.out()


def out2_rpb_case(epi):
    """RESID_GATE / ATTN_DO with out2 on a dense launch whose rows_per_batch (97) is not a multiple of 128: the gate row and the
    (b, s) of a token change inside a tile"""
    c = Checks()
    for bn in ((64, 128, 192, 256) if epi == EPI_RESID_GATE else (128, 256)):
        N = 512 if bn != 192 else 384
        if epi == EPI_RESID_GATE:
            probs = [_prob(4 * 97, N, 192, False, 1, epi=epi, bias=True, rows_per_batch=97, with_out2=True)]
            run(c, f"bn{bn}", probs, N, 192, trans_b=False, epi=epi, bn=bn)
        else:
            probs = [_prob(4 * 13, N, 192, True, 1, epi=epi, with_out2=True), _prob(4 * 97, N, 192, True, 11, epi=epi, with_out2=True, shift=1.0)]
            probs[0].update(rows_per_batch=13, s_offset=0)
            probs[1].update(rows_per_batch=97, s_offset=13)
            run(c, f"bn{bn}", probs, N, 192, trans_b=True, epi=epi, alpha=0.5, bn=bn, attn=dict(B=4, H=N // 128, S=112))
    return c.out()


def ragged_case(epi):
    """a pad-to-max row group (row bands) next to a dense one: dead rows must come back as exact zeros, computed rows as dense"""
    from qflux_b200 import lib
    c = Checks()
    R, valid = 700, (700, 100, 0, 420)
    plan = lib.RowBands.plan(list(valid), R)
    bands = lib.RowBands(plan[0], plan[1], DEV)
    trans_b = epi == EPI_DGELU
    probs = [_prob(R * len(valid), 256, 192, trans_b, 1, epi=epi, bias=not trans_b, rows_per_batch=R, with_out2=epi == EPI_RESID_GATE),
             _prob(300, 256, 192, trans_b, 11, epi=epi, bias=not trans_b, rows_per_batch=100, with_out2=epi == EPI_RESID_GATE, shift=1.0)]
    probs[0]["bands"] = bands
    run(c, "ragged", probs, 256, 192, trans_b=trans_b, epi=epi, bn=128)
    c.res["dead_ranges"] = bands.host_dead
    return c.out()


CASES = {}
for _bn in (64, 128, 192, 256):
    for _epi, _tb in ((EPI_BIAS, False), (EPI_BIAS, True), (EPI_GELU, False), (EPI_RESID_GATE, False), (EPI_DGELU, True), (EPI_ADD, True)):
        CASES[f"{EPI_NAME[_epi]}_{'nn' if _tb else 'nt'}_bn{_bn}"] = (lambda e, t, b: lambda: epilogue_case(e, t, b))(_epi, _tb, _bn)
for _bn in (128, 256):
    CASES[f"attn_do_nn_bn{_bn}"] = (lambda b: lambda: epilogue_case(EPI_ATTN_DO, True, b))(_bn)
CASES.update({
    "add_alias_flux_single": add_alias_case,
    "lora_a2_col0_groups": lora_col0_case,
    "six_resid_gate_nt": lambda: six_case(EPI_RESID_GATE, False),
    "six_bias_nt": lambda: six_case(EPI_BIAS, False),
    "six_dgelu_nn": lambda: six_case(EPI_DGELU, True),
    "six_add_nn": lambda: six_case(EPI_ADD, True),
    "resid_gate_out2_rpb97": lambda: out2_rpb_case(EPI_RESID_GATE),
    "attn_do_out2_rpb97": lambda: out2_rpb_case(EPI_ATTN_DO),
    "ragged_resid_gate": lambda: ragged_case(EPI_RESID_GATE),
    "ragged_gelu": lambda: ragged_case(EPI_GELU),
    "ragged_dgelu": lambda: ragged_case(EPI_DGELU),
})

if __name__ == "__main__":
    main(CASES, os.path.abspath(__file__), "gemm_tile_check.log")
