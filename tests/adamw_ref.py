"""TEST INFRASTRUCTURE ONLY — the optimizer tail of a training step restated in fp64: `torch.nn.utils.clip_grad_norm_` followed by one
`torch.optim.AdamW.step`, and the per-element bounds the fused kernels (qfx.h qfx_fused_adamw / qfx_grad_finalize and their _det
variants) are held to.

  * clip_grad_norm_: total_norm = sqrt(sum g^2), coef = min(1, max_norm / (total_norm + 1e-6)); max_norm <= 0 means no clip here
    (the kernels' convention).  The kernels see g = grad * pre_scale (1 / world, 1 / accumulated micro-steps).
  * AdamW.step (decoupled decay): p *= 1 - lr wd; m.lerp_(g, 1 - beta1); v = beta2 v + (1 - beta2) g^2;
    p -= (lr / bc1) m / (sqrt(v) / sqrt(bc2) + eps), bc_i = 1 - beta_i^step, eps outside the sqrt.
  * qfx.h: m and v are fp32, the new parameter is rounded to bf16 once.

Two modes give the step's scalars:
  torch  Python doubles, as torch computes them;
  abi    every scalar rounded to fp32, as the C ABI receives it, and 1 - beta, 1 - lr wd, bc1 = 1 - powf(beta1, step) and
         sqrtf(1 - powf(beta2, step)) formed in fp32 as qfx_fused_adamw forms them on the host.
They differ: at beta2 = 0.9999 the fp32 sqrt(bc2) is off by up to ~1e-4 relative in the first steps.  The fine bound is taken against
abi; torch gets the fixed allowances TORCH_MV_REL / TORCH_P_REL on top.

Bounds (`check_step`), each from the kernel's own state before the step:
  m, v   |kernel - ref| <= MV_ULPS fp32 eps of |beta m| + |(1 - beta) g| (v: of g^2), plus COEF_ULPS (v: twice that) of the gradient
         term when the clip is active (the kernels form the clip coefficient with --use_fast_math sqrtf and division);
  p      equal to bf16_rn(p64), except where p64 lies within W = P_WINDOW |update| + 2^-23 (|p_old| + |p64|) of a rounding midpoint;
         in general the bf16 rounding of some value in [p64 - W, p64 + W] (one ulp next to a midpoint; where p_old and the update
         cancel to a result far below both, W spans several ulps of that result).  |update| is taken with |beta1 m| + |(1 - beta1) g| in place of m:
         where the two terms of m cancel, m's own fp32 rounding is large next to m, and the update inherits it;
  stats  the flip count and the signed mean error in bf16 ulps, next to the same mean for the ideal rounding bf16_rn(p64): a
         systematic slip (eps, a bias correction, the decay) moves the first away from the second.
"""
from __future__ import annotations

import math

import numpy as np
import torch

EPS32 = 2.0 ** -23
MV_ULPS = 4
COEF_ULPS = 4
P_WINDOW = 1e-5
TORCH_MV_REL = 2e-4   # fp32(beta2 = 0.9999) moves 1 - beta2 by 1.66e-4 relative
TORCH_P_REL = 3e-4    # sqrt(bc2) in fp32 is off by up to ~1.1e-4 relative at beta2 = 0.9999 (steps 2-3); bc1, lr, eps far less
F64 = torch.float64


def clip_coef(sumsq, max_norm):
    """torch.nn.utils.clip_grad_norm_'s coefficient from the squared total norm; max_norm <= 0: no clip"""
    if max_norm <= 0:
        return 1.0
    return min(1.0, max_norm / (math.sqrt(sumsq) + 1e-6))


def _f32(x):
    return np.float32(x)


def scalars(mode, lr, beta1, beta2, eps, weight_decay, step, pre_scale=1.0, max_norm=0.0):
    """The step's scalars in `mode` ("torch" or "abi"), as Python floats."""
    if mode == "torch":
        return dict(lr=lr, b1=beta1, b2=beta2, omb1=1 - beta1, omb2=1 - beta2, eps=eps, decay=1 - lr * weight_decay,
                    step_size=lr / (1 - beta1 ** step), bc2_sqrt=(1 - beta2 ** step) ** 0.5, pre_scale=pre_scale, max_norm=max_norm)
    assert mode == "abi", mode
    lr32, b1, b2, eps32, wd = (_f32(x) for x in (lr, beta1, beta2, eps, weight_decay))
    one = _f32(1.0)
    powf = lambda b: _f32(float(b) ** step)  # glibc powf: the fp32 rounding of the exact power
    bc1, bc2 = one - powf(b1), one - powf(b2)
    return dict(lr=float(lr32), b1=float(b1), b2=float(b2), omb1=float(one - b1), omb2=float(one - b2), eps=float(eps32),
                decay=float(_f32(1.0 - float(lr32) * float(wd))),  # 1.f - lr * wd, contracted to one fma
                step_size=float(lr32) / float(bc1), bc2_sqrt=float(np.sqrt(bc2)), pre_scale=float(_f32(pre_scale)),
                max_norm=float(_f32(max_norm)))


def step_ref(p, g, m, v, S, sumsq=None):
    """One clip + AdamW step in fp64 from (p, g, m, v) (any float tensors of one shape) with the scalars S of `scalars()`.
    sumsq: the squared norm of grad * pre_scale the clip uses (default: fp64 over g, which must then be the whole flat gradient).
    Returns fp64 tensors p (before rounding), m, v, the magnitudes behind m and v, |update|, the update with |beta1 m| + |(1 - beta1) g|
    in place of m (what the rounding of m scales with where its two terms cancel), and the clip coefficient."""
    g, m, v, w = g.to(F64), m.to(F64), v.to(F64), p.to(F64)
    gs = g * S["pre_scale"]
    if sumsq is None:
        sumsq = float((gs * gs).sum())
    c = clip_coef(sumsq, S["max_norm"])
    gc = gs * c
    m1 = S["b1"] * m + S["omb1"] * gc
    v1 = S["b2"] * v + S["omb2"] * gc * gc
    den = v1.sqrt() / S["bc2_sqrt"] + S["eps"]
    upd = S["step_size"] * m1 / den
    p1 = w * S["decay"] - upd
    m_mag = (S["b1"] * m).abs() + (S["omb1"] * gc).abs()
    return dict(p=p1, m=m1, v=v1, m_mag=m_mag, v_mag=S["b2"] * v + S["omb2"] * gc * gc, m_term=(S["omb1"] * gc).abs(),
                v_term=S["omb2"] * gc * gc, upd=upd.abs(), upd_mag=S["step_size"] * m_mag / den, coef=c, clipped=c < 1.0, sumsq=sumsq)


def bf16_neighbour(r, x):
    """the bf16 value next to r (bf16 tensor) on the side of x (fp64 tensor); r itself where x == r"""
    b = r.contiguous().view(torch.int16).to(torch.int32)
    mag, sign = b & 0x7FFF, b & 0x8000
    rd = r.to(F64)
    away = x.abs() > rd.abs()
    sign = torch.where(mag == 0, torch.where(x < 0, 0x8000, 0), sign)
    mag2 = torch.where(x == rd, mag, torch.where(away, mag + 1, mag - 1))
    out = (sign | mag2)
    out = torch.where(out >= 0x8000, out - 0x10000, out).to(torch.int16)
    return out.view(torch.bfloat16)


def param_stats(p_new, p64, w_old, upd, window_rel=P_WINDOW):  # upd: the update's magnitude the window scales with
    """p_new (bf16) against bf16_rn(p64): flips, flips the window does not allow, signed mean errors"""
    p64 = p64.to(F64)
    r = p64.to(torch.bfloat16)
    nb = bf16_neighbour(r, p64)
    rd, nbd, pk = r.to(F64), nb.to(F64), p_new.to(F64)
    ulp = (nbd - rd).abs()
    ulp = torch.where(ulp == 0, torch.ldexp(torch.ones_like(rd), (torch.frexp(rd.abs().clamp_min(2.0 ** -126))[1] - 8)), ulp)
    window = window_rel * upd + 2.0 ** -23 * (w_old.to(F64).abs() + p64.abs())
    # allowed: the bf16 rounding of any value within the window of p64 (one ulp next to a midpoint; more where p_old and the
    # update cancel and the window spans several ulps of the small result)
    lo, hi = (p64 - window).to(torch.bfloat16).to(F64), (p64 + window).to(torch.bfloat16).to(F64)
    flip = pk != rd
    bad = flip & ((pk < lo) | (pk > hi))
    n = p64.numel()
    e, e0 = (pk - p64) / ulp, (rd - p64) / ulp
    return dict(n=n, flips=int(flip.sum()), flip_frac=float(flip.sum()) / max(n, 1), bad=int(bad.sum()),
                flip_ulps=float(((pk - rd).abs() / ulp).sum()),
                mean_err_ulps=float(e.mean()) if n else 0.0, ideal_mean_err_ulps=float(e0.mean()) if n else 0.0,
                max_err_ulps=float(e.abs().max()) if n else 0.0)


def check_step(before, after, hp, step, sumsq_k, mode="abi", tag=""):
    """before / after: dict(p, g, m, v) flat tensors (p bf16, gradient the whole flat buffer's elements the tensors use, m / v fp32).
    hp: dict(lr, beta1, beta2, eps, weight_decay, pre_scale, max_norm).  sumsq_k: the kernel's squared norm (the clip the kernel
    applied).  Returns (stats, failures) for one step in `mode`."""
    S = scalars(mode, hp["lr"], hp["beta1"], hp["beta2"], hp["eps"], hp["weight_decay"], step, hp["pre_scale"], hp["max_norm"])
    R = step_ref(before["p"], before["g"], before["m"], before["v"], S, sumsq=sumsq_k)
    clip = 1.0 if R["clipped"] else 0.0
    extra_mv = TORCH_MV_REL if mode == "torch" else 0.0
    fail = []
    st = {}
    for k, mag, term, cu in (("m", R["m_mag"], R["m_term"], COEF_ULPS), ("v", R["v_mag"], R["v_term"], 2 * COEF_ULPS)):
        err = (after[k].to(F64) - R[k]).abs()
        bound = EPS32 * (MV_ULPS * mag + clip * cu * term) + extra_mv * mag
        ulps = err / (EPS32 * mag).clamp_min(1e-300)
        st[f"{k}_max_ulps"] = float(torch.where(mag > 0, ulps, err * 0).max()) if err.numel() else 0.0
        nbad = int((err > bound).sum())
        if nbad:
            fail.append(f"{tag}{mode} step {step}: {k} beyond its bound at {nbad} elements (worst {st[f'{k}_max_ulps']:.1f} fp32 ulps)")
    ps = param_stats(after["p"], R["p"], before["p"], R["upd_mag"], P_WINDOW + (TORCH_P_REL if mode == "torch" else 0.0))
    st.update(ps)
    if ps["bad"]:
        fail.append(f"{tag}{mode} step {step}: {ps['bad']} parameters differ from bf16_rn(p64) away from a rounding midpoint")
    # the signed mean may differ from the ideal rounding's by at most the flips' own size (ulps) / n
    if abs(ps["mean_err_ulps"] - ps["ideal_mean_err_ulps"]) > ps["flip_ulps"] / max(ps["n"], 1) + 1e-12:
        fail.append(f"{tag}{mode} step {step}: signed mean error {ps['mean_err_ulps']:.3e} ulps vs {ps['ideal_mean_err_ulps']:.3e} ideal")
    st["clipped"] = bool(R["clipped"])
    return st, fail


# ------------------------------------------------------------------------------------------------ the kernel in fp32, for the CPU
MUTATIONS = ("none", "no_weight_decay", "no_bias_correction", "step_off_by_one", "eps_inside_sqrt", "bc2_without_sqrt",
             "clip_ignored")


def kernel_fp32(p, g, m, v, hp, step, sumsq, mutation="none"):
    """fused_adamw_kernel's arithmetic in fp32 on the CPU (exact sqrt / division; the GPU build uses the fast-math ones), with the
    abi scalars, optionally with one deliberate mistake.  p bf16, g / m / v fp32 (updated in place); returns the new bf16 p."""
    st = step + 1 if mutation == "step_off_by_one" else step
    S = scalars("abi", hp["lr"], hp["beta1"], hp["beta2"], hp["eps"], hp["weight_decay"], st, hp["pre_scale"], hp["max_norm"])
    f = lambda x: torch.tensor(x, dtype=torch.float32)
    coef = f(S["pre_scale"])
    if S["max_norm"] > 0 and mutation != "clip_ignored":
        c = f(S["max_norm"]) / (torch.sqrt(f(sumsq)) + f(1e-6))
        coef = coef * torch.clamp(c, max=1.0)
    bc1 = 1.0 - float(_f32(float(_f32(hp["beta1"])) ** st))
    bc2 = float(_f32(1.0) - _f32(float(_f32(hp["beta2"])) ** st))
    bc2s = float(np.sqrt(_f32(bc2)))
    if mutation == "no_bias_correction":
        bc1, bc2, bc2s = 1.0, 1.0, 1.0
    if mutation == "bc2_without_sqrt":
        bc2s = bc2
    step_size = f(S["lr"]) / f(bc1)
    gi = g * coef
    w = p.float()
    if mutation != "no_weight_decay":
        w = w * f(S["decay"])
    m.copy_(f(S["b1"]) * m + f(S["omb1"]) * gi)
    v.copy_(f(S["b2"]) * v + f(S["omb2"]) * gi * gi)
    if mutation == "eps_inside_sqrt":
        den = torch.sqrt(v / f(bc2) + f(S["eps"]))
    else:
        den = torch.sqrt(v) / f(bc2s) + f(S["eps"])
    return (w - step_size * m / den).to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------ schedules
def cosine_warmup(opt, warmup=5, total=20):
    """diffusers.optimization.get_scheduler("cosine", num_warmup_steps=warmup, num_training_steps=total) (num_cycles = 0.5), the
    configs' `scheduler_type: cosine`: lr 0 at the first step, linear warm-up, then half a cosine."""
    def f(step):
        if step < warmup:
            return step / max(1, warmup)
        prog = (step - warmup) / max(1, total - warmup)
        return max(0.0, 0.5 * (1.0 + math.cos(math.pi * 0.5 * 2.0 * prog)))
    return torch.optim.lr_scheduler.LambdaLR(opt, f)
