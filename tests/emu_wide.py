"""TEST INFRASTRUCTURE ONLY — CPU emulation of `qfx_lora_wgrad_tc` at every rank the kernel takes (1 <= r <= 128), installed on top of
tests/emu_lib.py for the wide-rank tests.

A group's columns of B are Rp = 64 * ceil(r / 64) wide (the LoRA rank padded to one or two 64-wide k-blocks).  For r <= 64 this is
emu_lib.lora_wgrad_tc exactly.  tools/wide_rank_check.py holds the kernel itself to fp64 bounds at these ranks on the GPU."""
from __future__ import annotations

import torch

import emu_lib


def lora_wgrad_tc(A, B, G_list, gs_i, gs_j, r, mode=0, Dg=0):
    Af, Bf = A.float(), B.float()
    rp = 64 * -(-r // 64)
    for g, G in enumerate(G_list):
        a = Af[:, g * Dg:(g + 1) * Dg] if mode == 1 else Af
        res = a.t() @ Bf[:, g * rp: g * rp + r]
        view = torch.as_strided(G, (res.shape[0], r), (gs_i, gs_j))
        view += res


def install(lib_module, base=None):
    """Install `base` (emu_lib.install by default; det_ref.install also works) over `qflux_b200.lib`, then the wide-rank
    lora_wgrad_tc over it and over emu_lib (which det_ref's lora_wgrad_tc_det calls).  Returns a callable that restores both."""
    restore_base = (base or emu_lib.install)(lib_module)
    saved_emu = emu_lib.lora_wgrad_tc
    emu_lib.lora_wgrad_tc = lora_wgrad_tc
    lib_module.lora_wgrad_tc = lora_wgrad_tc

    def restore():
        emu_lib.lora_wgrad_tc = saved_emu
        restore_base()
    return restore
