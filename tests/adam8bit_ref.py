"""TEST INFRASTRUCTURE ONLY — the 8-bit Adam of the reference's configs (`optimizer.class_path: bitsandbytes.optim.Adam8bit`), restated
in plain PyTorch, and the CPU emulation of `qflux_b200.lib.fused_adam8bit`.

  * `create_dynamic_map` restates bitsandbytes/functional.py `create_dynamic_map(signed, max_exponent_bits=7, total_bits=8)`: for each
    exponent i < 7 the means of a float32 `linspace(0.1, 1, ...)` scaled by 10^(i - 6) (2^i of them per sign when signed, 2^(i+1)
    unsigned), then 0 and 1.0, sorted.
  * `Adam8bit` restates bitsandbytes/optim/adam.py `Adam8bit` (an `Optimizer2State` "adam" with optim_bits 8, optim/optimizer.py) with
    percentile_clipping 100 and block-wise states, per parameter tensor in the parameter's flat row-major order:
      - numel < min_8bit_size: fp32 state1 / state2 (functional.py `optimizer_update_32bit`, csrc/kernels.cu `kOptimizer32bit2State`);
      - else uint8 state1 / state2, fp32 absmax1 / absmax2 per BLOCK elements, qmap1 / qmap2 = the signed / unsigned dynamic maps
        (functional.py `optimizer_update_8bit_blockwise`, kernels.cu `kOptimizerStatic8bit2StateBlockwise`): dequantize with the old
        absmax, update in fp32, new absmax = the block's max |s|, the parameter from the unquantized states, then each state stored as
        the nearest map entry to s / absmax (a tie takes the lower code) with the sign rule for state1.  A block whose absmax is 0
        stores the maps' zero codes (127 / 0, qfx.h QFX_ADAM8BIT_CODE*_ZERO).
    The scalars are formed in fp32 as the kernels form them; the parameter is rounded to its dtype after the step and again after the
    weight decay (when weight_decay > 0).  It computes in fp32 from `p.grad` of any dtype; bitsandbytes reads bf16 `.grad`s.
    One known difference: bitsandbytes' kernel pads the partial last block of state1 with code 128 (the smallest positive entry,
    5.5e-7), so a partial block whose real elements are all far below that fraction of the old absmax gets a tiny non-zero absmax
    there; here, as in the fused kernel, only the block's own elements count.
  * `fused_adam8bit` emulates the entry point of the same name over the flat buffers for `-m "not gpu"` runs (`install`), with the
    clip of qfx_fused_adamw in fp32.  tools/adam8bit_check.py holds the kernel to this restatement on the GPU.
"""
from __future__ import annotations

import numpy as np
import torch

import emu_lib

BLOCK = 256
CODE1_ZERO, CODE2_ZERO = 127, 0


def create_dynamic_map(signed=True, max_exponent_bits=7, total_bits=8):
    data, non_sign_bits = [], total_bits - 1
    for i in range(max_exponent_bits):
        items = int(2 ** (i + non_sign_bits - max_exponent_bits) + 1 if signed else 2 ** (i + non_sign_bits - max_exponent_bits + 1) + 1)
        b = torch.linspace(0.1, 1, items, dtype=torch.float32)
        means = (b[:-1] + b[1:]) / 2.0
        data += ((10 ** (-(max_exponent_bits - 1) + i)) * means).tolist()
        if signed:
            data += (-(10 ** (-(max_exponent_bits - 1) + i)) * means).tolist()
    data += [0, 1.0]
    data += [0] * (2 ** total_bits - len(data))
    return torch.tensor(sorted(data), dtype=torch.float32)


def scalars(lr, beta1, beta2, eps, weight_decay, step):
    """The kernels' fp32 scalars: correction2 * eps, step_size = -lr * correction2 / correction1, the decay factor."""
    f = np.float32
    lr, beta1, beta2, eps, weight_decay = f(lr), f(beta1), f(beta2), f(eps), f(weight_decay)
    c1 = f(1) - f(float(beta1) ** step)
    c2 = f(np.sqrt(f(1) - f(float(beta2) ** step)))
    step_size = -lr * c2 / c1
    decay = f(1) - lr * weight_decay if weight_decay > 0 else f(1)
    return dict(beta1=float(beta1), beta2=float(beta2), c2eps=float(c2 * eps), step_size=float(step_size), decay=float(decay))


def _t(x):
    return torch.tensor(x, dtype=torch.float32)


def quantize(q, x):
    """The nearest entry of the sorted map q to each x; a tie takes the lower code."""
    lo = (torch.searchsorted(q, x, right=True) - 1).clamp(0, 255)
    hi = (lo + 1).clamp(max=255)
    return torch.where((lo < 255) & (x > _t(0.5) * (q[lo] + q[hi])), hi, lo)


def update(p, g, s1_old, s2_old, sc, blockwise):
    """One step of one tensor on flat views: p (param dtype), g fp32, the dequantized old states fp32.  Returns (new parameter values,
    s1, s2) with s1 / s2 unquantized fp32."""
    b1, b2 = _t(sc["beta1"]), _t(sc["beta2"])
    finite = torch.isfinite(g)
    g = torch.where(finite, g, torch.zeros_like(g))
    s1 = s1_old * b1 + (_t(1) - b1) * g
    s2 = s2_old * b2 + ((_t(1) - b2) * g * g if blockwise else (_t(1) - b2) * (g * g))
    s1, s2 = torch.where(finite, s1, torch.zeros_like(s1)), torch.where(finite, s2, torch.zeros_like(s2))
    w = (p.float() + _t(sc["step_size"]) * (s1 / (s2.sqrt() + _t(sc["c2eps"])))).to(p.dtype)
    w = (w.float() * _t(sc["decay"])).to(p.dtype)
    return torch.where(finite, w, p), s1, s2


def block_absmax(s):
    n = s.numel()
    return torch.cat([s.abs(), s.new_zeros((-n) % BLOCK)]).view(-1, BLOCK).amax(1)


def quantize_states(s1, s2, absmax1, absmax2, q1, q2):
    """uint8 codes of the new states against the new per-block absmax (qfx.h's rule, bitsandbytes' sign rule for state1)."""
    n = s1.numel()
    a1, a2 = absmax1.repeat_interleave(BLOCK)[:n], absmax2.repeat_interleave(BLOCK)[:n]
    c1 = quantize(q1, s1 / a1)
    c1 = c1 + torch.where(torch.signbit(q1[c1]) != torch.signbit(s1), torch.where(s1 > 0, 1, -1), 0)
    c1 = torch.where(a1 > 0, c1, CODE1_ZERO)
    c2 = torch.where(a2 > 0, quantize(q2, s2 / a2), CODE2_ZERO)
    return c1.to(torch.uint8), c2.to(torch.uint8)


def step_tensor(p, g, st, sc, q1, q2):
    """bitsandbytes' update of one parameter: p a flat view (updated in place), g fp32 flat, st the tensor's state dict (updated)."""
    blockwise = "absmax1" in st
    if blockwise:
        n = p.numel()
        o1 = q1[st["state1"].long()] * st["absmax1"].repeat_interleave(BLOCK)[:n]
        o2 = q2[st["state2"].long()] * st["absmax2"].repeat_interleave(BLOCK)[:n]
    else:
        o1, o2 = st["state1"], st["state2"]
    w, s1, s2 = update(p, g, o1, o2, sc, blockwise)
    p.copy_(w)
    if blockwise:
        st["absmax1"], st["absmax2"] = block_absmax(s1), block_absmax(s2)
        st["state1"], st["state2"] = quantize_states(s1, s2, st["absmax1"], st["absmax2"], q1, q2)
    else:
        st["state1"], st["state2"] = s1, s2


class Adam8bit(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, optim_bits=32, args=None,
                 min_8bit_size=4096, percentile_clipping=100, block_wise=True, is_paged=False):
        if amsgrad or percentile_clipping != 100 or not block_wise or args is not None:
            raise NotImplementedError("the restatement covers amsgrad=False, percentile_clipping=100, block-wise states, args=None")
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay))
        self.min_8bit_size = min_8bit_size

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            for p in group["params"]:
                if p.grad is None:
                    continue
                st = self.state[p]
                if not st:
                    st["step"] = 0
                    if p.numel() < self.min_8bit_size:
                        st["state1"] = torch.zeros(p.numel(), dtype=torch.float32, device=p.device)
                        st["state2"] = torch.zeros(p.numel(), dtype=torch.float32, device=p.device)
                    else:
                        nb = -(-p.numel() // BLOCK)
                        st["state1"] = torch.zeros(p.numel(), dtype=torch.uint8, device=p.device)
                        st["state2"] = torch.zeros(p.numel(), dtype=torch.uint8, device=p.device)
                        st["absmax1"] = torch.zeros(nb, dtype=torch.float32, device=p.device)
                        st["absmax2"] = torch.zeros(nb, dtype=torch.float32, device=p.device)
                        st["qmap1"] = create_dynamic_map(True).to(p.device)
                        st["qmap2"] = create_dynamic_map(False).to(p.device)
                st["step"] += 1
                sc = scalars(group["lr"], group["betas"][0], group["betas"][1], group["eps"], group["weight_decay"], st["step"])
                flat = p.data.view(-1)
                step_tensor(flat, p.grad.float().reshape(-1), st, sc, st.get("qmap1"), st.get("qmap2"))
        return loss


def clip_coef(g, max_norm):
    """qfx_fused_adamw's clip coefficient on a flat fp32 gradient, in fp32 (1 when max_norm <= 0)."""
    if max_norm <= 0:
        return np.float32(1)
    f = np.float32
    c = f(max_norm) / (f(np.sqrt(f(float((g.double() ** 2).sum())))) + f(1e-6))
    return min(c, f(1))


# ---------------------------------------------------------------------------------------------------- emulation of lib.fused_adam8bit
def fused_adam8bit(tables, state_offsets, grad, state1, state2, absmax1, absmax2, s1_32, s2_32, qmap1, qmap2, sumsq, scratch, pre_scale,
                   max_norm, lr, beta1, beta2, eps, weight_decay, step, min_8bit_size):
    from qflux_b200 import lib
    assert step >= 1 and lr >= 0, "qfx_fused_adam8bit refuses step < 1 and lr < 0"
    assert scratch.dtype == torch.float32 and scratch.numel() >= lib.DET_NORM_PARTIALS
    assert state1.dtype == state2.dtype == torch.uint8 and state_offsets.dtype == torch.int64
    members, _ = tables
    g = grad * np.float32(pre_scale)
    sumsq.copy_((g.double() ** 2).sum().float().reshape(1))
    g = g * torch.tensor(clip_coef(g, max_norm), dtype=torch.float32)
    sc = scalars(lr, beta1, beta2, eps, weight_decay, step)
    for (p, off), so in zip(members, state_offsets.tolist()):
        n = p.numel()
        flat = p.reshape(-1).clone()
        if n >= min_8bit_size:
            nb = -(-n // BLOCK)
            st = dict(state1=state1[off: off + n], state2=state2[off: off + n], absmax1=absmax1[so: so + nb], absmax2=absmax2[so: so + nb])
            step_tensor(flat, g[off: off + n], st, sc, qmap1, qmap2)
            state1[off: off + n], state2[off: off + n] = st["state1"], st["state2"]
            absmax1[so: so + nb], absmax2[so: so + nb] = st["absmax1"], st["absmax2"]
        else:
            st = dict(state1=s1_32[so: so + n], state2=s2_32[so: so + n])
            step_tensor(flat, g[off: off + n], st, sc, qmap1, qmap2)
            s1_32[so: so + n], s2_32[so: so + n] = st["state1"], st["state2"]
        p.copy_(flat.view(p.shape))


_NAMES = ["fused_adam8bit"]


def install(lib_module):
    """emu_lib.install plus the 8-bit Adam entry point; returns the restore callable."""
    restore_emu = emu_lib.install(lib_module)
    saved = {n: getattr(lib_module, n) for n in _NAMES}
    for n in _NAMES:
        setattr(lib_module, n, globals()[n])

    def restore():
        for n, f in saved.items():
            setattr(lib_module, n, f)
        restore_emu()
    return restore
