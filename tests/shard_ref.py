"""TEST INFRASTRUCTURE ONLY — the sharded optimizer's entry points of `qflux_b200.lib` (qfx.h "slice forms", qfx_lora_pack / unpack) in
plain PyTorch for `-m "not gpu"` runs, installed on top of tests/dp_ref.py, tests/prodigy_ref.py and tests/adam8bit_ref.py.

Each slice form runs, on its chunks, the elementwise arithmetic of the emulation of its replicated entry point, with the clip taken from
the given sumsq, so a slice's elements come out with the bits the replicated emulation gives them when the clip factor is the same.
Prodigy's global sums are formed as the kernels form them: one fp64 partial per chunk, added by the scalar kernel's fixed order
(thread t takes chunks t, t + 256, ..., then the 256 sums in thread order).  `fused_prodigy` (the replicated entry point) is replaced by
the same per-chunk form, so the replicated and sharded emulations share one order, as the kernels do.
tests/test_sharded_optimizer.py holds the kernels to fp64 / exact restatements on the GPU.
"""
from __future__ import annotations

import math

import numpy as np
import torch

import adam8bit_ref
import dp_ref
import prodigy_ref

BF = torch.bfloat16


def _chunks(members):
    from qflux_b200 import lib
    return [(i, e) for i, (p, _) in enumerate(members) for e in range(0, p.numel(), lib.ADAMW_CHUNK)]


def _pieces(tables, chunk_range, g_lo=None, g_hi=None):
    """(member index, param, grad offset, e0, e1) per chunk of the range, clipped to the gradient range [g_lo, g_hi)."""
    from qflux_b200 import lib
    members, _ = tables
    out = []
    for i, e in _chunks(members)[chunk_range[0]: chunk_range[1]]:
        p, off = members[i]
        e0, e1 = e, min(p.numel(), e + lib.ADAMW_CHUNK)
        if g_lo is not None:
            e0, e1 = max(e0, g_lo - off), min(e1, g_hi - off)
        if e1 > e0:
            out.append((i, p, off, e0, e1))
    return out


def _write(p, e0, new):
    flat = p.reshape(-1).clone()
    flat[e0: e0 + new.numel()] = new
    p.copy_(flat.view(p.shape))


def _f32(x):
    return float(torch.tensor(x, dtype=torch.float32))


def sumsq_det(x, pre_scale, out, *, scratch):
    from qflux_b200 import lib
    assert scratch.numel() >= lib.DET_NORM_PARTIALS and x.dtype == torch.float32
    out.copy_(((x * _f32(pre_scale)) ** 2).sum().reshape(1))


def fused_adamw_slice(tables, chunk_range, state_base, grad, exp_avg, exp_avg_sq, sumsq, pre_scale, max_norm, lr, beta1, beta2, eps,
                      weight_decay, step):
    """emu_lib.fused_adamw's arithmetic on the slice."""
    pre_scale, max_norm, lr, beta1, beta2, eps, weight_decay = (_f32(x) for x in (pre_scale, max_norm, lr, beta1, beta2, eps, weight_decay))
    coef = min(1.0, max_norm / (float(sumsq.sqrt()) + 1e-6)) if max_norm > 0 else 1.0
    bc1, bc2 = _f32(1 - _f32(beta1 ** step)), _f32(1 - _f32(beta2 ** step))
    omb1, omb2, decay = _f32(1 - beta1), _f32(1 - beta2), _f32(1 - lr * weight_decay)
    for _, p, off, e0, e1 in _pieces(tables, chunk_range):
        gi = (grad[off + e0: off + e1] * pre_scale) * coef
        sl = slice(off + e0 - state_base, off + e1 - state_base)
        m, v = exp_avg[sl], exp_avg_sq[sl]
        w = p.reshape(-1)[e0:e1].float() * decay
        m.mul_(beta1).add_(gi, alpha=omb1)
        v.mul_(beta2).addcmul_(gi, gi, value=omb2)
        _write(p, e0, (w - (lr / bc1) * m / (v.sqrt() / _f32(bc2 ** 0.5) + eps)).to(BF))


def fused_adam8bit_slice(tables, chunk_range, state_base, state_offsets, grad, state1, state2, absmax1, absmax2, s1_32, s2_32, qmap1,
                         qmap2, sumsq, pre_scale, max_norm, lr, beta1, beta2, eps, weight_decay, step, min_8bit_size):
    """adam8bit_ref.fused_adam8bit's arithmetic on the slice (the clip coefficient from sumsq)."""
    f = np.float32
    coef = f(1)
    if max_norm > 0:
        coef = min(f(max_norm) / (f(np.sqrt(f(float(sumsq)))) + f(1e-6)), f(1))
    sc = adam8bit_ref.scalars(lr, beta1, beta2, eps, weight_decay, step)
    so_all = state_offsets.tolist()
    B = adam8bit_ref.BLOCK
    for i, p, off, e0, e1 in _pieces(tables, chunk_range):
        g = (grad[off + e0: off + e1] * f(pre_scale)) * torch.tensor(coef, dtype=torch.float32)
        flat = p.reshape(-1)[e0:e1].clone()
        so, s = so_all[i], slice(off + e0 - state_base, off + e1 - state_base)
        if p.numel() >= min_8bit_size:
            a = slice(so + e0 // B, so + -(-e1 // B))
            st = dict(state1=state1[s], state2=state2[s], absmax1=absmax1[a], absmax2=absmax2[a])
            adam8bit_ref.step_tensor(flat, g, st, sc, qmap1, qmap2)
            state1[s], state2[s], absmax1[a], absmax2[a] = st["state1"], st["state2"], st["absmax1"], st["absmax2"]
        else:
            st = dict(state1=s1_32[so + e0: so + e1], state2=s2_32[so + e0: so + e1])
            adam8bit_ref.step_tensor(flat, g, st, sc, qmap1, qmap2)
            s1_32[so + e0: so + e1], s2_32[so + e0: so + e1] = st["state1"], st["state2"]
        _write(p, e0, flat)


# ---- Prodigy, per chunk
def _pass_a(tables, chunk_range, state_base, grad, exp_avg, exp_avg_sq, s, p0, scalars, coef, pre_scale, lr, beta1, beta2, beta3,
            weight_decay, decouple, use_bias_correction, safeguard_warmup, d0):
    """prodigy_ref.fused_prodigy's first loop, per chunk; returns the chunks' (dot, sum |s|)."""
    from qflux_b200 import lib
    sc = scalars.tolist()
    d, k = sc[lib.PRODIGY_D], sc[lib.PRODIGY_K]
    bc = math.sqrt(1 - beta2 ** (k + 1)) / (1 - beta1 ** (k + 1)) if use_bias_correction else 1.0
    dlr = d * lr * bc
    wd_coupled = 0.0 if decouple else weight_decay
    parts = []
    for _, p, off, e0, e1 in _pieces(tables, chunk_range):
        sl = slice(off + e0 - state_base, off + e1 - state_base)
        w = p.reshape(-1)[e0:e1].float()
        gi = grad[off + e0: off + e1] * pre_scale * coef + wd_coupled * w
        dot = float((gi.double() * (p0[sl].double() - w.double())).sum())
        exp_avg[sl] = beta1 * exp_avg[sl] + d * (1 - beta1) * gi if beta1 > 0 else gi
        exp_avg_sq[sl] = beta2 * exp_avg_sq[sl] + d * d * (1 - beta2) * gi * gi
        s[sl] = beta3 * s[sl] + d / d0 * (d if safeguard_warmup else dlr) * gi
        parts.append((dot, float(s[sl].double().abs().sum())))
    return parts


def _scalar(scalars, part, lr, beta1, beta2, beta3, use_bias_correction, d0, d_coef, growth_rate):
    """prodigy_scalar_kernel: the partials in its fixed order, then the update of d, d_max, d_num, k."""
    from qflux_b200 import lib
    part = part.reshape(-1, 2).tolist()
    threads = [[0.0, 0.0] for _ in range(256)]
    for c, (a, b) in enumerate(part):
        threads[c % 256][0] += a
        threads[c % 256][1] += b
    dot = den = 0.0
    for a, b in threads:
        dot += a
        den += b
    sc = scalars.tolist()
    d = sc[lib.PRODIGY_D]
    k = sc[lib.PRODIGY_K]
    bc = math.sqrt(1 - beta2 ** (k + 1)) / (1 - beta1 ** (k + 1)) if use_bias_correction else 1.0
    dlr = d * lr * bc
    d_num = beta3 * sc[lib.PRODIGY_D_NUM] + d / d0 * dlr * dot
    sc[lib.PRODIGY_DLR] = dlr
    if den == 0:
        sc[lib.PRODIGY_SKIPPED] = 1.0
        scalars.copy_(torch.tensor(sc, dtype=torch.float64))
        return False
    d_hat = d_coef * d_num / den
    if d == d0:
        d = max(d, d_hat)
    d_max = max(sc[lib.PRODIGY_D_MAX], d_hat)
    d = min(d_max, d * growth_rate)
    sc[lib.PRODIGY_D], sc[lib.PRODIGY_D_MAX], sc[lib.PRODIGY_D_NUM] = d, d_max, d_num
    sc[lib.PRODIGY_K] += 1
    sc[lib.PRODIGY_SKIPPED], sc[lib.PRODIGY_D_DEN], sc[lib.PRODIGY_D_HAT] = 0.0, den, d_hat
    scalars.copy_(torch.tensor(sc, dtype=torch.float64))
    return True


def _pass_b(tables, chunk_range, state_base, exp_avg, exp_avg_sq, scalars, beta1, eps, weight_decay, decouple):
    from qflux_b200 import lib
    sc = scalars.tolist()
    d, dlr = sc[lib.PRODIGY_D], sc[lib.PRODIGY_DLR]
    wd_decoupled = weight_decay if decouple else 0.0
    ms = 1.0 if beta1 > 0 else d
    for _, p, off, e0, e1 in _pieces(tables, chunk_range):
        sl = slice(off + e0 - state_base, off + e1 - state_base)
        w = p.reshape(-1)[e0:e1].float()
        _write(p, e0, (w - dlr * (wd_decoupled * w + ms * exp_avg[sl] / (exp_avg_sq[sl].sqrt() + d * eps))).to(BF))


def _coef(sumsq, max_norm):
    return min(1.0, max_norm / (math.sqrt(float(sumsq)) + 1e-6)) if max_norm > 0 else 1.0


def fused_prodigy(tables, grad, exp_avg, exp_avg_sq, s, p0, scalars, sumsq, scratch, pre_scale, max_norm, lr, beta1, beta2, beta3, eps,
                  weight_decay, decouple, use_bias_correction, safeguard_warmup, d0, d_coef, growth_rate):
    """The replicated entry point with the kernels' per-chunk partials (prodigy_ref's arithmetic otherwise)."""
    assert lr > 0 and d0 > 0 and scratch.numel() >= prodigy_ref.prodigy_scratch_floats(tables)
    g = grad * pre_scale
    sumsq.copy_((g * g).sum().reshape(1))
    full = (0, len(_chunks(tables[0])))
    parts = _pass_a(tables, full, 0, grad, exp_avg, exp_avg_sq, s, p0, scalars, _coef(sumsq, max_norm), pre_scale, lr, beta1, beta2,
                    beta3, weight_decay, decouple, use_bias_correction, safeguard_warmup, d0)
    if _scalar(scalars, torch.tensor(parts, dtype=torch.float64), lr, beta1, beta2, beta3, use_bias_correction, d0, d_coef, growth_rate):
        _pass_b(tables, full, 0, exp_avg, exp_avg_sq, scalars, beta1, eps, weight_decay, decouple)


def prodigy_slice_partials(tables, chunk_range, state_base, grad, exp_avg, exp_avg_sq, s, p0, scalars, sumsq, part, pre_scale, max_norm,
                           lr, beta1, beta2, beta3, weight_decay, decouple, use_bias_correction, safeguard_warmup, d0):
    assert lr > 0 and d0 > 0 and part.dtype == torch.float64
    parts = _pass_a(tables, chunk_range, state_base, grad, exp_avg, exp_avg_sq, s, p0, scalars, _coef(sumsq, max_norm), pre_scale, lr,
                    beta1, beta2, beta3, weight_decay, decouple, use_bias_correction, safeguard_warmup, d0)
    if parts:
        part.reshape(-1, 2)[chunk_range[0]: chunk_range[1]] = torch.tensor(parts, dtype=torch.float64)


def prodigy_slice_update(tables, chunk_range, state_base, n_grad, exp_avg, exp_avg_sq, scalars, part, lr, beta1, beta2, beta3, eps,
                         weight_decay, decouple, use_bias_correction, d0, d_coef, growth_rate):
    if _scalar(scalars, part, lr, beta1, beta2, beta3, use_bias_correction, d0, d_coef, growth_rate):
        _pass_b(tables, chunk_range, state_base, exp_avg, exp_avg_sq, scalars, beta1, eps, weight_decay, decouple)


def lora_pack(tables, chunk_range, g_lo, g_hi, flat):
    assert flat.dtype == BF and flat.numel() >= g_hi - g_lo
    for _, p, off, e0, e1 in _pieces(tables, chunk_range, g_lo, g_hi):
        flat[off + e0 - g_lo: off + e1 - g_lo] = p.reshape(-1)[e0:e1]


def lora_unpack(tables, chunk_range, g_lo, g_hi, flat):
    assert flat.dtype == BF and flat.numel() >= g_hi - g_lo
    for _, p, off, e0, e1 in _pieces(tables, chunk_range, g_lo, g_hi):
        _write(p, e0, flat[off + e0 - g_lo: off + e1 - g_lo])


_NAMES = ["sumsq_det", "fused_adamw_slice", "fused_adam8bit_slice", "fused_prodigy", "prodigy_slice_partials", "prodigy_slice_update",
          "lora_pack", "lora_unpack", "fused_adam8bit", "prodigy_scratch_floats"]
_FROM = {"fused_adam8bit": adam8bit_ref, "prodigy_scratch_floats": prodigy_ref}


def install(lib_module):
    """dp_ref.install (emu_lib, the deterministic and the data-parallel entry points) plus the optimizers' entry points above;
    returns the restore callable."""
    restore_dp = dp_ref.install(lib_module)
    saved = {n: getattr(lib_module, n) for n in _NAMES}
    for n in _NAMES:
        setattr(lib_module, n, getattr(_FROM[n], n) if n in _FROM else globals()[n])

    def restore():
        for n, f in saved.items():
            setattr(lib_module, n, f)
        restore_dp()
    return restore
