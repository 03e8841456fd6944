"""TEST INFRASTRUCTURE ONLY — the deterministic entry points of `qflux_b200.lib` (`*_det`, picked under
torch.use_deterministic_algorithms(True)) in plain PyTorch for `-m "not gpu"` runs.

Each computes what emu_lib.py's emulation of the entry point it is named after computes (a CPU sum is already reproducible), after
checking that the fp32 scratch the host hands over satisfies qfx.h's size rule, which the kernels enforce too.  tools/determinism_check.py
holds the kernels themselves to fp64 bounds and to bitwise repeats on the GPU.
"""
from __future__ import annotations

import torch

import emu_lib


def _need(scratch, n):
    assert scratch.dtype == torch.float32 and scratch.is_contiguous() and scratch.numel() >= n, (scratch.numel(), n)


def attn_bwd_det(Q, K, V, dO, lse, delta, dQ_accum, dK, dV, kv_len=None, scale=None, txt_len=None, split=0):
    emu_lib.attn_bwd(Q, K, V, dO, lse, delta, dQ_accum, dK, dV, kv_len=kv_len, scale=scale, txt_len=txt_len, split=split)


def lora_wgrad_tc_det(A, B, G_list, gs_i, gs_j, r, mode=0, Dg=0, *, scratch):
    from qflux_b200 import lib
    _need(scratch, lib.det_scratch_wgrad_tc(A.shape[0], A.shape[1], 1 if mode == 1 else len(G_list), r))
    emu_lib.lora_wgrad_tc(A, B, G_list, gs_i, gs_j, r, mode=mode, Dg=Dg)


def lora_wgrad_det(P, Q, G, gs_i, gs_j, r, *, scratch):
    from qflux_b200 import lib
    _need(scratch, lib.det_scratch_wgrad(P.shape[0], P.shape[1], r))
    emu_lib.lora_wgrad(P, Q, G, gs_i, gs_j, r)


def mod_grad_det(g, rows_per_batch, sum_out=None, m=None, prod_out=None, mean=None, rstd=None, *, scratch):
    from qflux_b200 import lib
    _need(scratch, lib.det_scratch_mod_grad(g.shape[0], rows_per_batch, g.shape[1]))
    emu_lib.mod_grad(g, rows_per_batch, sum_out=sum_out, m=m, prod_out=prod_out, mean=mean, rstd=rstd)


def flow_loss_det(pred, x0, noise, w, norm, loss, dpred=None, grad_scale=1.0, *, scratch):
    from qflux_b200 import lib
    _need(scratch, lib.DET_LOSS_PARTIALS)
    emu_lib.flow_loss(pred, x0, noise, w, norm, loss, dpred, grad_scale)


def grad_finalize_det(g_f32, pre_scale, max_norm, sumsq, out_bf16, *, scratch):
    from qflux_b200 import lib
    _need(scratch, lib.DET_NORM_PARTIALS)
    emu_lib.grad_finalize(g_f32, pre_scale, max_norm, sumsq, out_bf16)


def fused_adamw_det(tables, grad, exp_avg, exp_avg_sq, sumsq, pre_scale, max_norm, lr, beta1, beta2, eps, weight_decay, step, *, scratch):
    from qflux_b200 import lib
    _need(scratch, lib.DET_NORM_PARTIALS)
    emu_lib.fused_adamw(tables, grad, exp_avg, exp_avg_sq, sumsq, pre_scale, max_norm, lr, beta1, beta2, eps, weight_decay, step)


_NAMES = ["attn_bwd_det", "lora_wgrad_tc_det", "lora_wgrad_det", "mod_grad_det", "flow_loss_det", "grad_finalize_det", "fused_adamw_det"]


def install(lib_module):
    """emu_lib.install plus the deterministic entry points; returns the restore callable."""
    restore_emu = emu_lib.install(lib_module)
    saved = {n: getattr(lib_module, n) for n in _NAMES}
    g = globals()
    for n in _NAMES:
        setattr(lib_module, n, g[n])

    def restore():
        for n, f in saved.items():
            setattr(lib_module, n, f)
        restore_emu()
    return restore
