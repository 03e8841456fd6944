"""GPU check of the HBM-bound glue entry points the training step calls (stream-pair LayerNorm-modulate, q/k-norm + RoPE, attention
delta, flow-matching input, add, timestep embedding, zero_rows) through the C ABI, each against

  (a) an independent fp64 restatement of the reference semantics (oracle RMSNorm conventions, F.layer_norm, RoPE, diffusers'
      timestep embedding, fp64 autograd for the backward kernels), next to the same reference evaluated in bf16 on the device
      ("bf16 eager"), which calibrates what close means;
  (b) tests/emu_lib.py on CPU copies of the same inputs — the emulation the CPU suite runs the fused model on.

Errors are measured per row group and per row: the second group's operands are chosen far from the first group's, so a row that
uses the wrong group's modulation vector, norm weight, sample length or joint offset is off by O(1) in that row alone.

Emulator fidelity (b) is element-wise:
  * data movement (V / dV copies, dO scatter, control copy, padding, add, gate multiply, the flow-matching mix): bit-identical;
  * values rounded to bf16 at the kernel's documented rounding points: |kernel - emu| <= the rounding-flip bound.  Kernel and
    emulation reduce in a different order, so a rounded intermediate v can land on the neighbouring bf16 value: it moves by at
    most ulp(v), and that move reaches the output scaled by the local gain of the ops after it; the output's own rounding adds
    one ulp(out).  Each case spells out its bound from the kernel's rounding points;
  * fp32 reductions: |kernel - emu| <= 1e-5 * sum|terms| per element.
Each case returns a dict of measurements plus `fail`, the list of violated checks (empty = pass).  Run stand-alone:
`python tools/glue_check.py [case ...]` (one subprocess per case).
"""
import math
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from harness import ROOT, main  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

BF, F64 = torch.bfloat16, torch.float64
EPS = 1e-6
RED_TOL = 1e-5   # fp32 reductions, relative to sum |terms|
ROW_FLOOR = 1e-3  # per-row / per-group allowance above 1.25x the bf16-eager error


def _mk(*shape, scale=1.0, seed=0, dtype=BF, device="cuda", shift=0.0):
    g = torch.Generator(device=device).manual_seed(seed)
    return (torch.randn(*shape, device=device, generator=g) * scale + shift).to(dtype)


def ulp_bf16(v):
    """spacing of bf16 at |v| (fp64 tensor); subnormal/zero values get the smallest normal spacing"""
    v = v.double().abs().clamp_min(2.0 ** -126)
    _, e = torch.frexp(v)
    return torch.ldexp(torch.ones_like(v), (e - 8).to(torch.int32))


def row_rel(a, ref):
    """per-row relative L2 of 2-D a vs ref (fp64)"""
    a, ref = a.double().flatten(1), ref.double().flatten(1)
    return (a - ref).norm(dim=1) / (ref.norm(dim=1) + 1e-30)


def rel(a, ref):
    a, ref = a.double(), ref.double()
    return ((a - ref).norm() / (ref.norm() + 1e-30)).item()


class Checks:
    """collects measurements and violated checks of one case"""

    def __init__(self):
        self.res, self.fail = {}, []

    def check(self, ok, what):
        if not bool(ok):
            self.fail.append(what)

    def vs_refs(self, name, k, f64, eager, groups):
        """kernel / bf16-eager error vs fp64, globally, per row group and per row (rows = dim 0 of 2-D views)"""
        for gname, sl in groups:
            ke, ee = rel(k[sl], f64[sl]), rel(eager[sl], f64[sl])
            kr, er = row_rel(k[sl], f64[sl]).max().item(), row_rel(eager[sl], f64[sl]).max().item()
            self.res[f"{name}_{gname}"] = [ke, ee]
            self.res[f"{name}_{gname}_rowmax"] = [kr, er]
            self.check(ke < 5e-3 and ke <= 1.25 * ee + ROW_FLOOR, f"{name}_{gname}: kernel {ke:.2e} vs bf16 eager {ee:.2e}")
            self.check(kr < 2e-2 and kr <= 1.25 * er + ROW_FLOOR, f"{name}_{gname} row max: kernel {kr:.2e} vs bf16 eager {er:.2e}")

    def exact(self, name, k, ref):
        k, ref = k.cpu(), ref.cpu()
        same = (k.view(torch.int16) == ref.view(torch.int16)) if k.dtype == BF else (k == ref)
        self.res[f"{name}_bitfrac"] = same.double().mean().item() if same.numel() else 1.0
        self.check(bool(same.all()), f"{name}: not bit-identical ({int((~same).sum())} of {same.numel()} differ)")

    def emu_bound(self, name, k, e, bound):
        """bf16 results: |kernel - emu| <= bound (fp64 tensor, same shape) element-wise"""
        k, e = k.cpu().double(), e.cpu().double()
        d = (k - e).abs()
        self.res[f"emu_{name}_bitfrac"] = (d == 0).double().mean().item()
        self.res[f"emu_{name}_max_over_bound"] = (d / bound.cpu()).max().item()
        self.check(bool((d <= bound.cpu()).all()), f"emu_{name}: {int((d > bound.cpu()).sum())} elements beyond the rounding-flip bound")

    def emu_red(self, name, k, e, mag):
        """fp32 reduction results: |kernel - emu| <= RED_TOL * mag (sum of |terms|) element-wise"""
        k, e, mag = k.cpu().double(), e.cpu().double(), mag.cpu().double()
        d = (k - e).abs()
        self.res[f"emu_{name}_bitfrac"] = (d == 0).double().mean().item()
        self.res[f"emu_{name}_max_rel"] = (d / (mag + 1e-30)).max().item()
        self.check(bool((d <= RED_TOL * mag + 1e-30).all()), f"emu_{name}: fp32 reduction beyond {RED_TOL} relative")

    def out(self):
        self.res["fail"] = self.fail
        return self.res


def _up(v):  # ulp of a rounded intermediate, taken at the larger end of its binade so a flip across a binade edge is covered
    return ulp_bf16(v.double().abs() * (1 + 2.0 ** -7))


# ============================================================================ fp64 references (device-agnostic; checked on CPU too)
def ln_mod_ref(x, sh_rows, sc_rows, eps=EPS):
    """LayerNorm (no affine) + AdaLN modulate, per-row shift/scale [M, D]"""
    return F.layer_norm(x, (x.shape[1],), eps=eps) * (1 + sc_rows) + sh_rows


def rms_ref(x, w, eps=EPS):
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * w


def rope_ref(x, cs):
    """x [..., 128]; cs [..., 64, 2] (cos, sin) broadcastable; pairs (2i, 2i+1), like apply_rotary_emb_qwen / _real"""
    a, b = x.unflatten(-1, (64, 2)).unbind(-1)
    c, s = cs[..., 0], cs[..., 1]
    return torch.stack([a * c - b * s, a * s + b * c], -1).flatten(-2)


def rope_rows(rope, B, n, off):
    """rope table rows of positions [off, off + n) as [B, n, 1, 64, 2]"""
    r = rope[off:off + n][None].expand(B, n, 64, 2) if rope.dim() == 3 else rope[:, off:off + n]
    return r[:, :, None]


def timestep_ref(t, dim, scale):
    """diffusers get_timestep_embedding(flip_sin_to_cos=True, downscale_freq_shift=0, scale), fp64"""
    half = dim // 2
    arg = scale * t.double()[:, None] * torch.exp(-math.log(10000.0) * torch.arange(half, dtype=F64, device=t.device) / half)[None]
    return torch.cat([arg.cos(), arg.sin()], -1), torch.cat([arg, arg], -1)


def flow_rule(x0, noise, sigma):
    """the kernel's stated rounding rule: bf16( bf16(bf16(1 - s) * x0) + bf16(s * noise) ),  s = bf16(sigma)"""
    s = sigma.to(BF).float().view(-1, *([1] * (x0.dim() - 1)))
    one_m = (1 - s).to(BF).float()
    return ((one_m * x0.float()).to(BF).float() + (s * noise.float()).to(BF).float()).to(BF)


def _groups(split, M):
    return (("g0", slice(0, split)), ("g1", slice(split, M)))


# ============================================================================ LayerNorm + modulate (stream pair)
def _ln_operands(D, T, L, B, device):
    M, split = B * (T + L), B * T
    x = _mk(M, D, seed=1, scale=2.0, shift=0.5, device=device)
    mod = torch.cat([_mk(B, 6 * D, seed=2, scale=0.3, device=device),  # group 0 (text): small shift/scale/gate
                     _mk(B, 6 * D, seed=3, scale=0.3, device=device)], 1)
    off = torch.zeros(12 * D, device=device)
    off[6 * D:7 * D], off[7 * D:8 * D], off[8 * D:9 * D] = 4.0, 2.0, -3.0  # group 1 (image): far from group 0
    mod = (mod.float() + off).to(BF)
    sh = (mod[:, 0:D], mod[:, 6 * D:7 * D])  # strided [B, D] views of one [B, 12D] tensor (ld = 12D), as the model passes them
    sc = (mod[:, D:2 * D], mod[:, 7 * D:8 * D])
    gt = (mod[:, 2 * D:3 * D], mod[:, 8 * D:9 * D])
    rows = lambda v: torch.cat([v[0].repeat_interleave(T, 0), v[1].repeat_interleave(L, 0)])
    return x, sh, sc, gt, rows, M, split


def ln_mod_pair(D, T=7, L=33, B=3):
    from qflux_b200 import lib
    import emu_lib as emu
    c = Checks()
    x, sh, sc, gt, rows, M, split = _ln_operands(D, T, L, B, "cuda")
    grp = _groups(split, M)
    y = torch.empty_like(x)
    mean, rstd = torch.empty(M, device="cuda"), torch.empty(M, device="cuda")
    lib.ln_modulate_fwd_pair(x, y, (sh[0], sc[0], T), (sh[1], sc[1], L), split, mean, rstd)
    # (a) fp64 and bf16 eager (the reference's own expression on bf16 operands)
    xd = x.double().requires_grad_(True)
    y64 = ln_mod_ref(xd, rows(sh).double(), rows(sc).double())
    xb = x.clone().requires_grad_(True)
    yb = F.layer_norm(xb, (D,), eps=EPS) * (1 + rows(sc)) + rows(sh)
    c.vs_refs("fwd", y, y64.detach(), yb.detach(), grp)
    mu64, rs64 = x.double().mean(1), torch.rsqrt(x.double().var(1, unbiased=False) + EPS)
    c.res["mean_max_abs_over_mean_abs_x"] = ((mean.double() - mu64).abs() / x.double().abs().mean(1)).max().item()
    c.res["rstd_max_rel"] = ((rstd.double() - rs64).abs() / rs64).max().item()
    c.check(c.res["mean_max_abs_over_mean_abs_x"] < RED_TOL and c.res["rstd_max_rel"] < RED_TOL, "mean / rstd vs fp64")
    # (b) emulation on CPU
    xc = x.cpu()
    ye, me, re_ = torch.empty_like(xc), torch.empty(M), torch.empty(M)
    emu.ln_modulate_fwd_pair(xc, ye, (sh[0].cpu(), sc[0].cpu(), T), (sh[1].cpu(), sc[1].cpu(), L), split, me, re_)
    xf = xc.float()
    n = ((xf - me[:, None]) * re_[:, None]).to(BF).double()          # rounding point 1: bf16(LN(x))
    scb = (1 + rows(sc).cpu().float()).to(BF).double()                # bf16(1 + scale): same operands, no reduction -> no flip
    m = (n * scb).to(BF).double()                                     # rounding point 2
    bound = _up(n) * scb.abs() + _up(m) + _up(torch.maximum(ye.double().abs(), y.cpu().double().abs()))
    c.emu_bound("ln_fwd", y, ye, bound)
    c.emu_red("ln_mean", mean, me, xf.abs().mean(1))
    c.emu_red("ln_rstd", rstd, re_, re_.abs())
    # ---- backward, with and without dres and the gates
    dy, dres = _mk(M, D, seed=4), _mk(M, D, seed=5)
    (g64,) = torch.autograd.grad(y64, xd, dy.double())
    (gb,) = torch.autograd.grad(yb, xb, dy)
    for with_res in (False, True):
        for with_gate in (False, True):
            tag = f"bwd{'_res' if with_res else ''}{'_gate' if with_gate else ''}"
            dx = torch.empty_like(x)
            dxg = torch.empty_like(x) if with_gate else None
            lib.ln_modulate_bwd_pair(dy, x, mean, rstd, (sc[0], T, gt[0] if with_gate else None), (sc[1], L, gt[1] if with_gate else None),
                                     split, dx, dres=dres if with_res else None, dx_gated=dxg)
            dx64 = g64 + (dres.double() if with_res else 0)
            dxb = (dres + gb) if with_res else gb  # bf16 eager: autograd's bf16 grad, then the bf16 residual add
            c.vs_refs(tag, dx, dx64, dxb, grp)
            if with_gate:
                c.vs_refs(tag + "_gated", dxg, dx64 * rows(gt).double(), dxb * rows(gt), grp)
            dxe = torch.empty_like(xc)
            dxge = torch.empty_like(xc) if with_gate else None
            emu.ln_modulate_bwd_pair(dy.cpu(), xc, mean.cpu(), rstd.cpu(), (sc[0].cpu(), T, gt[0].cpu() if with_gate else None),
                                     (sc[1].cpu(), L, gt[1].cpu() if with_gate else None), split, dxe,
                                     dres=dres.cpu() if with_res else None, dx_gated=dxge)
            # bound: g = bf16(dy * bf16(1 + scale)) is exact-input (no flip); d = bf16(rstd * (g - s1 - xh * s2)) with fp32
            # row sums s1, s2 in a different order -> pre-rounding difference <= rstd * (2^-22 (|g|+|s1|+|xh s2|) + RED_TOL
            # (mean|g| + |xh| mean|g xh|)) plus one flip of d; o = bf16(dres + d) adds one flip; dxg = bf16(o * gate) scales it.
            rs, mu = rstd.cpu().double()[:, None], mean.cpu().double()[:, None]
            g = (dy.cpu().float() * (1 + rows(sc).cpu().float()).to(BF).float()).to(BF).double()
            xh = (xc.double() - mu) * rs
            s1, s2 = g.mean(1, keepdim=True), (g * xh).mean(1, keepdim=True)
            d = (rs * (g - s1 - xh * s2)).to(BF).double()
            pre = rs * (2.0 ** -22 * (g.abs() + s1.abs() + (xh * s2).abs()) + RED_TOL * (g.abs().mean(1, keepdim=True) +
                                                                                        xh.abs() * (g * xh).abs().mean(1, keepdim=True)))
            bd = pre + _up(d)
            o = dxe.double()
            if with_res:
                bd = bd + _up(torch.maximum(o.abs(), dx.cpu().double().abs()))
            c.emu_bound(tag, dx, dxe, bd)
            if with_gate:
                gr = rows(gt).cpu().double()
                c.emu_bound(tag + "_gated", dxg, dxge, bd * gr.abs() + _up(torch.maximum(dxge.double().abs(), dxg.cpu().double().abs())))
    return c.out()


# ============================================================================ q/k RMSNorm + RoPE (stream pair)
def _qk_operands(H, T, L, B, per_sample, device):
    S, tokens, split = T + L, B * (T + L), B * T
    qkv = _mk(tokens, 3 * H * 128, seed=11, device=device)
    w = dict(q0=_mk(128, seed=12, scale=0.2, shift=1.0, device=device), k0=_mk(128, seed=13, scale=0.2, shift=1.0, device=device),
             q1=_mk(128, seed=14, scale=0.2, shift=-1.5, device=device), k1=_mk(128, seed=15, scale=0.2, shift=-1.5, device=device))
    g = torch.Generator(device=device).manual_seed(16)
    ang = torch.rand(*((B,) if per_sample else ()), S, 64, device=device, generator=g) * 6.28
    rope = torch.stack([ang.cos(), ang.sin()], -1).contiguous()  # [S,64,2] or [B,S,64,2] fp32
    return qkv, w, rope, S, tokens, split


def _qk_fwd_ref(qkv, w, rope, T, L, B, H, norm):
    """per group: (q, k, v) [B, n, H, 128] in the dtype of `qkv`'s math; norm(x, w) is the RMSNorm convention"""
    out = []
    for wq, wk, n, off, sl in ((w["q0"], w["k0"], T, 0, slice(0, B * T)), (w["q1"], w["k1"], L, T, slice(B * T, None))):
        x = qkv[sl].view(B, n, 3, H, 128)
        cs = rope_rows(rope, B, n, off).to(qkv.dtype if qkv.dtype == F64 else torch.float32)
        q = rope_ref(norm(x[:, :, 0], wq).to(cs.dtype), cs)
        k = rope_ref(norm(x[:, :, 1], wk).to(cs.dtype), cs)
        if qkv.dtype != F64:
            q, k = q.to(BF), k.to(BF)
        out.append((q, k, x[:, :, 2], n, off))
    return out


def _eager_norm(round_mid, device):
    """the reference's RMSNorm on bf16 operands: diffusers RMSNorm (Qwen, round_mid) or the torch.nn.RMSNorm module (FLUX)"""
    from oracle.mmdit_oracle import diffusers_rms_norm
    if round_mid:
        return lambda x, w: diffusers_rms_norm(x, w, EPS)

    def norm(x, w):  # one module per call: autograd keeps each group's weight
        mod = torch.nn.RMSNorm(128, eps=EPS, device=device, dtype=BF)
        with torch.no_grad():
            mod.weight.copy_(w)
        return mod(x)
    return norm


def _token_major(Qh, B, n, off):  # [B,H,S,128] -> [B*n, H*128] rows of the group at joint offset off
    return Qh[:, :, off:off + n].permute(0, 2, 1, 3).reshape(B * n, -1)


def qk_pair(H, T, L, B, round_mid, per_sample=False):
    from qflux_b200 import lib
    import emu_lib as emu
    c = Checks()
    qkv, w, rope, S, tokens, split = _qk_operands(H, T, L, B, per_sample, "cuda")
    c.res["tokens_x_H_mod_8"] = tokens * H % 8
    g0, g1 = (w["q0"], w["k0"], T, 0), (w["q1"], w["k1"], L, T)
    Q, K, V = (torch.zeros(B, H, S, 128, device="cuda", dtype=BF) for _ in range(3))
    lib.qk_norm_rope_fwd_pair(qkv, g0, g1, split, rope, Q, K, V, round_mid=round_mid)
    qd = qkv.double().requires_grad_(True)
    r64 = _qk_fwd_ref(qd, {k: v.double() for k, v in w.items()}, rope.double(), T, L, B, H, rms_ref)
    qb = qkv.clone().requires_grad_(True)
    rbf = _qk_fwd_ref(qb, w, rope, T, L, B, H, _eager_norm(round_mid, "cuda"))
    for (q64, k64, v64, n, off), (qe, ke, ve, _, _), gname in zip(r64, rbf, ("g0", "g1")):
        whole = (("all", slice(None)),)
        c.vs_refs(f"q_{gname}", _token_major(Q, B, n, off), q64.detach().reshape(B * n, -1), qe.detach().reshape(B * n, -1), whole)
        c.vs_refs(f"k_{gname}", _token_major(K, B, n, off), k64.detach().reshape(B * n, -1), ke.detach().reshape(B * n, -1), whole)
        c.exact(f"v_{gname}", _token_major(V, B, n, off), ve.detach().reshape(B * n, -1))
    # emulation (CPU)
    cpu = lambda g: (g[0].cpu(), g[1].cpu(), g[2], g[3])
    Qe, Ke, Ve = (torch.zeros(B, H, S, 128, dtype=BF) for _ in range(3))
    emu.qk_norm_rope_fwd_pair(qkv.cpu(), cpu(g0), cpu(g1), split, rope.cpu(), Qe, Ke, Ve, round_mid=round_mid)
    # bound: n = RMSNorm output rounded to bf16 (round_mid: bf16(bf16(x r) w), two rounding points) may flip by ulp(n)
    # (+ ulp(x r) |w|); RoPE mixes a pair with |cos|, |sin| <= 1, so the output moves by <= the pair's two flips + ulp(out)
    for which, (Kk, Ke_) in enumerate(((Q, Qe), (K, Ke))):
        bound = torch.zeros(B, H, S, 128, dtype=F64)
        for wq, wk, n, off, sl in ((w["q0"], w["k0"], T, 0, slice(0, split)), (w["q1"], w["k1"], L, T, slice(split, None))):
            f = qkv[sl].cpu().float().view(B, n, 3, H, 128)[:, :, which]
            ww = (wk if which else wq).cpu().float()
            r = torch.rsqrt(f.pow(2).mean(-1, keepdim=True) + EPS)
            mid = (f * r).to(BF).double()
            nn_ = (mid * ww.double()).to(BF).double() if round_mid else (f * r * ww).to(BF).double()
            dn = _up(nn_) + (_up(mid) * ww.double().abs() if round_mid else 0)
            dpair = dn.unflatten(-1, (64, 2)).sum(-1, keepdim=True).expand(*dn.shape[:-1], 64, 2).flatten(-2)
            bound[:, :, off:off + n] = dpair.permute(0, 2, 1, 3)
        big = torch.maximum(Kk.cpu().double().abs(), Ke_.double().abs())
        c.emu_bound("fwd_" + "qk"[which], Kk, Ke_, bound + _up(big))
    c.exact("emu_fwd_v", V, Ve)
    # ---- backward: fp64 autograd and bf16 eager autograd (which holds dQ in bf16), then clear_dq
    dQ = _mk(B, H, S, 128, seed=20, dtype=torch.float32)
    dK, dV = _mk(B, H, S, 128, seed=21), _mk(B, H, S, 128, seed=22)
    dqkv = torch.empty_like(qkv)
    dQ_keep = dQ.clone()
    lib.qk_norm_rope_bwd_pair(dQ, dK, dV, qkv, g0, g1, split, rope, dqkv, round_mid=round_mid)
    c.exact("bwd_dQ_untouched", dQ, dQ_keep)

    def cot(t, n, off, dt):
        return t[:, :, off:off + n].permute(0, 2, 1, 3).to(dt)
    outs64, cots64, outsb, cotsb = [], [], [], []
    for (q, k, v, n, off), (qe, ke, ve, _, _) in zip(r64, rbf):
        outs64 += [q, k, v]
        cots64 += [cot(dQ, n, off, F64), cot(dK, n, off, F64), cot(dV, n, off, F64)]
        outsb += [qe, ke, ve]
        cotsb += [cot(dQ, n, off, BF), cot(dK, n, off, BF), cot(dV, n, off, BF)]
    (d64,) = torch.autograd.grad(outs64, qd, cots64)
    (db,) = torch.autograd.grad(outsb, qb, cotsb)
    sl3 = lambda t, j: t.view(tokens, 3, -1)[:, j]
    grp = _groups(split, tokens)
    for j, nm in ((0, "dq"), (1, "dk")):
        c.vs_refs("bwd_" + nm, sl3(dqkv, j), sl3(d64, j), sl3(db, j), grp)
    c.exact("bwd_dv_copy", sl3(dqkv, 2), sl3(db, 2))
    # clear_dq: same dqkv bit for bit, dQ exactly zero afterwards (the two groups cover every joint position here)
    dQc, dqkv_c = dQ_keep.clone(), torch.empty_like(qkv)
    lib.qk_norm_rope_bwd_pair(dQc, dK, dV, qkv, g0, g1, split, rope, dqkv_c, round_mid=round_mid, clear_dq=True)
    c.exact("clear_dq_dqkv", dqkv_c, dqkv)
    c.check(bool((dQc == 0).all()), "clear_dq: dQ not all zero")
    # emulation of the backward
    dqkv_e = torch.empty_like(qkv, device="cpu")
    dQe = dQ_keep.cpu()
    emu.qk_norm_rope_bwd_pair(dQe, dK.cpu(), dV.cpu(), qkv.cpu(), cpu(g0), cpu(g1), split, rope.cpu(), dqkv_e, round_mid=round_mid,
                              clear_dq=True)
    c.check(bool((dQe == 0).all()), "emu clear_dq: dQ not all zero")
    # bound: gn = bf16(conj-rotated bf16 grad) may flip by ulp(gn); o = r gn w - f r^3 mean(gn w f), then one flip of o
    bnd = torch.zeros(tokens, 3, H, 128, dtype=F64)
    for wq, wk, n, off, sl in ((w["q0"], w["k0"], T, 0, slice(0, split)), (w["q1"], w["k1"], L, T, slice(split, None))):
        x = qkv[sl].cpu().double().view(B, n, 3, H, 128)
        cs = rope_rows(rope.cpu(), B, n, off).double()
        for which, (ww, gsrc) in enumerate(((wq, dQ_keep), (wk, dK))):
            go = gsrc[:, :, off:off + n].cpu().permute(0, 2, 1, 3).to(BF).double()
            gn = rope_ref(go, torch.stack([cs[..., 0], -cs[..., 1]], -1)).to(BF).double()
            f, wd = x[:, :, which], ww.cpu().double()
            r = torch.rsqrt(f.pow(2).mean(-1, keepdim=True) + EPS)
            ug = _up(gn)
            dot = (gn * wd * f).mean(-1, keepdim=True)
            b_ = r * wd.abs() * ug + f.abs() * r ** 3 * (ug * (wd * f).abs()).mean(-1, keepdim=True) + \
                2.0 ** -20 * (r * (gn * wd).abs() + f.abs() * r ** 2 * dot.abs())
            bnd[sl, which] = b_.reshape(B * n, H, 128)
    bnd = bnd.view(tokens, -1)
    big = torch.maximum(dqkv.cpu().double().abs(), dqkv_e.double().abs())
    bnd = bnd + _up(big)
    c.emu_bound("bwd_dqk", sl3(dqkv, slice(0, 2)).reshape(tokens, -1).cpu(), sl3(dqkv_e, slice(0, 2)).reshape(tokens, -1),
                bnd.view(tokens, 3, -1)[:, :2].reshape(tokens, -1))
    c.exact("emu_bwd_dv", sl3(dqkv, 2), sl3(dqkv_e, 2))
    return c.out()


def rmsnorm_convention(H=4, tokens=600):
    """Which rounding torch.nn.RMSNorm uses on CUDA for bf16 (FLUX's q/k norm) and diffusers RMSNorm (Qwen's): the kernel with an
    identity rotation emits the normalised values themselves; count the elements that differ from each module."""
    from qflux_b200 import lib
    from oracle.mmdit_oracle import diffusers_rms_norm
    c = Checks()
    qkv = _mk(tokens, 3 * H * 128, seed=31, scale=1.5)
    wq, wk = _mk(128, seed=32, scale=0.3, shift=1.0), _mk(128, seed=33, scale=0.3, shift=1.0)
    rope = torch.stack([torch.ones(tokens, 64, device="cuda"), torch.zeros(tokens, 64, device="cuda")], -1).contiguous()
    q_by = {}
    for rm in (False, True):
        Q, K, V = (torch.zeros(1, H, tokens, 128, device="cuda", dtype=BF) for _ in range(3))
        lib.qk_norm_rope_fwd_pair(qkv, (wq, wk, tokens, 0), (wq, wk, 1, 0), tokens, rope, Q, K, V, round_mid=rm)
        q_by[rm] = Q[0].permute(1, 0, 2).reshape(tokens, H * 128)
    x = qkv.view(tokens, 3, H, 128)[:, 0]
    mod = torch.nn.RMSNorm(128, eps=EPS, device="cuda", dtype=BF)
    with torch.no_grad():
        mod.weight.copy_(wq)
        ref_torch = mod(x).reshape(tokens, -1)
    ref_diff = diffusers_rms_norm(x, wq, EPS).reshape(tokens, -1)
    for rname, ref in (("torch_nn_RMSNorm_cuda", ref_torch), ("diffusers_RMSNorm_cuda", ref_diff)):
        for rm in (False, True):
            d = (q_by[rm].view(torch.int16) != ref.view(torch.int16)).double().mean().item()
            c.res[f"{rname}_vs_round_mid_{int(rm)}_differ_frac"] = d
    # the settings the models use: FLUX round_mid=0 against torch.nn.RMSNorm, Qwen round_mid=1 against diffusers RMSNorm
    t0, t1 = c.res["torch_nn_RMSNorm_cuda_vs_round_mid_0_differ_frac"], c.res["torch_nn_RMSNorm_cuda_vs_round_mid_1_differ_frac"]
    d0, d1 = c.res["diffusers_RMSNorm_cuda_vs_round_mid_0_differ_frac"], c.res["diffusers_RMSNorm_cuda_vs_round_mid_1_differ_frac"]
    c.check(t0 < t1 and t0 < 0.02, f"FLUX (round_mid=0) is not the torch.nn.RMSNorm convention on CUDA ({t0:.3f} vs {t1:.3f})")
    c.check(d1 < d0 and d1 < 0.02, f"Qwen (round_mid=1) is not the diffusers RMSNorm convention ({d1:.3f} vs {d0:.3f})")
    return c.out()


# ============================================================================ attention delta (stream pair)
def attn_delta_pair(H=3, T=7, L=34, B=3, gap=2, tail=3):
    from qflux_b200 import lib
    import emu_lib as emu
    c = Checks()
    tokens, split, S = B * (T + L), B * T, T + gap + L + tail
    O, dO = _mk(tokens, H * 128, seed=41), _mk(tokens, H * 128, seed=42)
    SENT_D, SENT_O = -7.25, 3.0
    delta = torch.full((B, H, S), SENT_D, device="cuda")
    dOj = torch.full((B, H, S, 128), SENT_O, device="cuda", dtype=BF)
    g0, g1 = (T, 0), (L, T + gap)
    lib.attn_delta_pair(O, dO, delta, g0, g1, split, dOj)
    de, dOje = torch.full((B, H, S), SENT_D), torch.full((B, H, S, 128), SENT_O, dtype=BF)
    emu.attn_delta_pair(O.cpu(), dO.cpu(), de, g0, g1, split, dOje)
    covered = torch.zeros(S, dtype=torch.bool)
    ref = torch.full((B, H, S), SENT_D, dtype=F64)
    mag = torch.ones(B, H, S, dtype=F64)
    refj = torch.full((B, H, S, 128), SENT_O, dtype=BF)
    for (n, off), sl in ((g0, slice(0, split)), (g1, slice(split, None))):
        o, g = O[sl].cpu().double().view(B, n, H, 128), dO[sl].cpu().double().view(B, n, H, 128)
        ref[:, :, off:off + n] = (o * g).sum(-1).permute(0, 2, 1)
        mag[:, :, off:off + n] = (o * g).abs().sum(-1).permute(0, 2, 1)
        refj[:, :, off:off + n] = dO[sl].cpu().view(B, n, H, 128).permute(0, 2, 1, 3)
        covered[off:off + n] = True
    d = (delta.cpu().double() - ref).abs()
    c.res["delta_max_rel_vs_fp64"] = (d / mag).max().item()
    c.check(bool((d <= RED_TOL * mag).all()), "delta vs fp64 row sums")
    for gname, (n, off) in (("g0", g0), ("g1", g1)):
        c.res[f"delta_{gname}_max_rel"] = (d[:, :, off:off + n] / mag[:, :, off:off + n]).max().item()
    c.exact("dO_joint", dOj, refj)
    c.check(bool((delta.cpu()[:, :, ~covered] == SENT_D).all()), "delta: uncovered positions lost the sentinel")
    c.res["uncovered_positions"] = int((~covered).sum())
    c.emu_red("delta", delta, de, mag)
    c.exact("emu_dO_joint", dOj, dOje)
    return c.out()


# ============================================================================ flow-matching input, add, timestep, zero_rows
def flow_input():
    from qflux_b200 import lib
    import emu_lib as emu
    c = Checks()
    B, Ltmax, Lcmax, Cc = 4, 37, 21, 64
    Lt_h, Lc_h = [Ltmax, 5, 17, 30], [3, 0, Lcmax, 11]
    Ltot = max(a + b for a, b in zip(Lt_h, Lc_h)) + 4
    x0, noise, ctrl = _mk(B, Ltmax, Cc, seed=51), _mk(B, Ltmax, Cc, seed=52), _mk(B, Lcmax, Cc, seed=53)
    sigma = torch.tensor([0.999, 0.5, 0.123, 0.0371], device="cuda")  # not bf16-representable: the sigma rounding matters
    Lt, Lc = torch.tensor(Lt_h, device="cuda", dtype=torch.int32), torch.tensor(Lc_h, device="cuda", dtype=torch.int32)
    packed = torch.full((B, Ltot, Cc), 9.0, device="cuda", dtype=BF)
    lib.flow_noisy_input_var(x0, noise, ctrl, sigma, Lt, Lc, packed)
    mix = flow_rule(x0, noise, sigma)
    pk = packed.cpu()
    for b in range(B):
        lt, lc = Lt_h[b], Lc_h[b]
        c.exact(f"var_noisy_b{b}", pk[b, :lt], mix[b, :lt])
        c.exact(f"var_control_b{b}", pk[b, lt:lt + lc], ctrl[b, :lc])
        c.exact(f"var_pad_b{b}", pk[b, lt + lc:], torch.zeros_like(pk[b, lt + lc:]))
    pe = torch.full((B, Ltot, Cc), 9.0, dtype=BF)
    emu.flow_noisy_input_var(x0.cpu(), noise.cpu(), ctrl.cpu(), sigma.cpu(), Lt.cpu(), Lc.cpu(), pe)
    c.exact("emu_var", packed, pe)
    # dense
    L, Lcd = 29, 13
    x0d, nd, cd = _mk(B, L, Cc, seed=54), _mk(B, L, Cc, seed=55), _mk(B, Lcd, Cc, seed=56)
    pd = torch.empty(B, L + Lcd, Cc, device="cuda", dtype=BF)
    lib.flow_noisy_input(x0d, nd, cd, sigma, pd)
    c.exact("dense_noisy", pd[:, :L], flow_rule(x0d, nd, sigma))
    c.exact("dense_control", pd[:, L:], cd)
    pde = torch.empty(B, L + Lcd, Cc, dtype=BF)
    emu.flow_noisy_input(x0d.cpu(), nd.cpu(), cd.cpu(), sigma.cpu(), pde)
    c.exact("emu_dense", pd, pde)
    return c.out()


def add():
    from qflux_b200 import lib
    import emu_lib as emu
    c = Checks()
    n = 64 * 256 * 3 + 77  # odd, and not a multiple of the kernel's grid stride (64 CTAs x 256 threads)
    a, b = _mk(n, seed=61, scale=3.0), _mk(n, seed=62)
    ref = (a.float() + b.float()).to(BF)
    out = torch.empty_like(a)
    lib.add_bf16(a, b, out)
    c.exact("add", out, ref)
    oe = torch.empty(n, dtype=BF)
    emu.add_bf16(a.cpu(), b.cpu(), oe)
    c.exact("emu_add", out, oe)
    a2 = a.clone()
    lib.add_bf16(a2, b, a2)  # out aliasing a, as flux_model.py accumulates temb
    c.exact("add_aliased", a2, ref)
    return c.out()


def timestep():
    """Qwen: scale 1000 on sigma rounded to bf16.  FLUX: scale 1 on bf16(bf16(t) * 1000), and the same for guidance (args to 3500 rad).
    Bound: one ulp of the bf16 output plus the fp32 argument error carried through |d cos| <= 1: the kernel forms
    scale * (t * exp(-ln(1e4) j / half)) in fp32 (a few ulp relative), and the approximate sin/cos of the fast-math build add an
    absolute error that grows with |arg| on top of a 2^-20 floor.  The 2^-20 |arg| coefficient rests on an H100 measurement
    (H100 80GB HBM3: worst element at half the bound; 4.6 ulps at 1000 rad, 13.9 ulps at 7500 rad)."""
    from qflux_b200 import lib
    import emu_lib as emu
    c = Checks()
    B, dim = 6, 256
    g = torch.Generator(device="cuda").manual_seed(71)
    u = torch.rand(B, device="cuda", generator=g)
    u[0], u[1] = 1.0, 0.0
    cases = dict(qwen=(u.to(BF).float(), 1000.0),
                 flux_t=((u.to(BF) * 1000).float(), 1.0),
                 flux_guidance=((torch.tensor([1.0, 2.5, 3.5, 4.0, 7.5, 3.5], device="cuda").to(BF) * 1000).float(), 1.0))
    for name, (t32, scale) in cases.items():
        out = torch.empty(B, dim, device="cuda", dtype=BF)
        lib.timestep_sinusoid(t32.contiguous(), scale, out)
        ref, arg = timestep_ref(t32.cpu(), dim, scale)
        bound = _up(ref) + 2.0 ** -20 * arg.abs() + 2.0 ** -20
        err = (out.cpu().double() - ref).abs()
        c.res[f"{name}_max_arg_rad"] = arg.abs().max().item()
        c.res[f"{name}_max_err_ulps"] = (err / ulp_bf16(ref)).max().item()
        c.res[f"{name}_max_err_over_bound"] = (err / bound).max().item()
        c.check(bool((err <= bound).all()), f"timestep {name}: beyond one ulp + argument-error bound")
        oe = torch.empty(B, dim, dtype=BF)
        emu.timestep_sinusoid(t32.cpu(), scale, oe)
        c.emu_bound(f"timestep_{name}", out, oe, 2 * bound)
    return c.out()


def zero_rows():
    from qflux_b200 import lib
    c = Checks()
    R, ld, ncols = 40, 136, 64
    buf = torch.full((R, ld), 5.5, device="cuda", dtype=BF)
    spans = [(2, 5), (9, 10), (17, 30)]
    ranges = torch.tensor(spans, device="cuda", dtype=torch.int32).reshape(-1)
    lib.zero_rows(buf, ncols, ranges, len(spans))
    ref = torch.full((R, ld), 5.5, dtype=BF)
    for lo, hi in spans:
        ref[lo:hi, :ncols] = 0
    c.exact("zero_rows", buf, ref)
    return c.out()


# ============================================================================ emulator fidelity of the remaining elementwise entry points
def emu_misc():
    from qflux_b200 import lib
    import emu_lib as emu
    c = Checks()
    M, D, rpb = 96, 512, 32
    a, gate = _mk(M, D, seed=81), _mk(M // rpb, 3 * D, seed=82)[:, D:2 * D]
    out = torch.empty_like(a)
    lib.gate_mul(a, gate, rpb, out)
    oe = torch.empty(M, D, dtype=BF)
    emu.gate_mul(a.cpu(), gate.cpu(), rpb, oe)
    c.exact("emu_gate_mul", out, oe)
    # rmsnorm_rows: n = bf16(x r) may flip, then one flip of y = bf16(n w)
    x, w = _mk(70, 3584, seed=83, scale=3.0), _mk(3584, seed=84, scale=0.2, shift=1.0)
    y, ye = torch.empty_like(x), torch.empty(70, 3584, dtype=BF)
    lib.rmsnorm_rows(x, w, y)
    emu.rmsnorm_rows(x.cpu(), w.cpu(), ye)
    xf = x.cpu().double()
    nrm = (xf * torch.rsqrt(xf.pow(2).mean(1, keepdim=True) + EPS)).to(BF).double()
    c.emu_bound("rmsnorm_rows", y, ye, _up(nrm) * w.cpu().double().abs() + _up(torch.maximum(y.cpu().double().abs(), ye.double().abs())))
    # mod_grad (fp32 column sums)
    g, m = _mk(M, D, seed=85), _mk(M, D, seed=86)
    mean, rstd = m.float().mean(1), torch.rsqrt(m.float().var(1, unbiased=False) + EPS)
    so, po = torch.zeros(M // rpb, D, device="cuda"), torch.zeros(M // rpb, D, device="cuda")
    lib.mod_grad(g, rpb, sum_out=so, m=m, prod_out=po, mean=mean, rstd=rstd)
    soe, poe = torch.zeros(M // rpb, D), torch.zeros(M // rpb, D)
    emu.mod_grad(g.cpu(), rpb, sum_out=soe, m=m.cpu(), prod_out=poe, mean=mean.cpu(), rstd=rstd.cpu())
    gv = g.cpu().double().view(-1, rpb, D)
    mh = ((m.cpu().float() - mean.cpu()[:, None]) * rstd.cpu()[:, None]).to(BF).double().view(-1, rpb, D)
    c.emu_red("mod_grad_sum", so, soe, gv.abs().sum(1))
    # the bf16 normalised m inside may flip (ulp(mh) |g|) besides the reduction order
    c.emu_red("mod_grad_prod", po, poe, (gv * mh).abs().sum(1) + (_up(mh) * gv.abs()).sum(1) / RED_TOL)
    # gemv_act: bf16 SiLU input (exact-input -> may flip across the fast-math exp), fp32 dot, one flip of y
    xs, W, bias = _mk(3, 1024, seed=87), _mk(640, 1024, seed=88, scale=0.02), _mk(640, seed=89)
    yg, yge = torch.empty(3, 640, device="cuda", dtype=BF), torch.empty(3, 640, dtype=BF)
    lib.gemv_act(xs, W, bias, yg, 1)
    emu.gemv_act(xs.cpu(), W.cpu(), bias.cpu(), yge, 1)
    si = F.silu(xs.cpu().float()).to(BF).double()
    mag = si.abs() @ W.cpu().double().abs().t() + (_up(si) @ W.cpu().double().abs().t()) / RED_TOL
    c.emu_bound("gemv_act", yg, yge, RED_TOL * mag + _up(torch.maximum(yg.cpu().double().abs(), yge.double().abs())))
    # flow_loss: loss is an fp32 reduction, dpred one rounding of an fp32 product chain
    B, L, Cc = 2, 40, 64
    x0, noise, pred = _mk(B, L, Cc, seed=90), _mk(B, L, Cc, seed=91), _mk(B, 2 * L, Cc, seed=92)
    wt = torch.rand(B, L, device="cuda") + 0.5
    norm = 1.0 / (B * L * Cc)
    loss, dpred = torch.zeros(1, device="cuda"), torch.empty_like(pred)
    lib.flow_loss(pred, x0, noise, wt, norm, loss, dpred)
    le, dpe = torch.zeros(1), torch.empty(B, 2 * L, Cc, dtype=BF)
    emu.flow_loss(pred.cpu(), x0.cpu(), noise.cpu(), wt.cpu(), norm, le, dpe)
    c.emu_red("flow_loss", loss, le, le.abs())
    c.emu_bound("flow_dpred", dpred, dpe, _up(torch.maximum(dpred.cpu().double().abs(), dpe.double().abs())))
    # lora_wgrad (fp32 atomics)
    P, Qm = _mk(300, 256, seed=93), _mk(300, 64, seed=94)
    G, Ge = torch.zeros(256, 16, device="cuda"), torch.zeros(256, 16)
    lib.lora_wgrad(P, Qm, G, 16, 1, 16)
    emu.lora_wgrad(P.cpu(), Qm.cpu(), Ge, 16, 1, 16)
    c.emu_red("lora_wgrad", G, Ge, P.cpu().double().abs().t() @ Qm.cpu().double()[:, :16].abs())
    # grad_finalize: fp32 sum of squares, clipped bf16 cast
    gg = _mk(5000, seed=95, dtype=torch.float32)
    ss, ob = torch.zeros(1, device="cuda"), torch.empty(5000, device="cuda", dtype=BF)
    lib.grad_finalize(gg, 0.5, 1.0, ss, ob)
    sse, obe = torch.zeros(1), torch.empty(5000, dtype=BF)
    emu.grad_finalize(gg.cpu(), 0.5, 1.0, sse, obe)
    c.emu_red("grad_sumsq", ss, sse, sse.abs())
    c.emu_bound("grad_clip_cast", ob, obe, RED_TOL * obe.double().abs() + _up(torch.maximum(ob.cpu().double().abs(), obe.double().abs())))
    return c.out()


CASES = {}
for _D in (256, 512, 1024, 2048, 3072, 4096):
    CASES[f"ln_mod_pair_D{_D}"] = (lambda D: lambda: ln_mod_pair(D, T=7, L=33, B=3))(_D)           # M = 120, split = 21
    CASES[f"ln_mod_pair_D{_D}_oddM"] = (lambda D: lambda: ln_mod_pair(D, T=7, L=34, B=3))(_D)      # M = 123: surplus rows
for _rm in (0, 1):
    for _ps in (0, 1):
        CASES[f"qk_pair_h2_rm{_rm}_rope{'B' if _ps else 'S'}"] = (lambda rm, ps: lambda: qk_pair(2, 7, 34, 3, bool(rm), bool(ps)))(_rm, _ps)
        CASES[f"qk_pair_h24_rm{_rm}_rope{'B' if _ps else 'S'}"] = (lambda rm, ps: lambda: qk_pair(24, 40, 97, 2, bool(rm), bool(ps)))(_rm, _ps)
CASES.update({
    "rmsnorm_convention": rmsnorm_convention,
    "attn_delta_pair": attn_delta_pair,
    "attn_delta_pair_h24": lambda: attn_delta_pair(H=24, T=40, L=97, B=2, gap=5, tail=1),
    "flow_input": flow_input,
    "add_bf16": add,
    "timestep": timestep,
    "zero_rows": zero_rows,
    "emu_misc": emu_misc,
})

if __name__ == "__main__":
    main(CASES, os.path.abspath(__file__), "glue_check.log")
