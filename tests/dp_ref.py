"""TEST INFRASTRUCTURE ONLY — `qflux_b200.lib.dp_reduce_det` (the fixed-order data-parallel gradient sum) in plain PyTorch for
`-m "not gpu"` runs, installed on top of tests/emu_lib.py and tests/det_ref.py.  tests/test_dp_determinism.py holds the kernel to the
same sequential fp32 sum on the GPU.
"""
from __future__ import annotations

import torch

import det_ref


def dp_reduce_det(srcs, dst):
    """qfx_dp_reduce_det: a sequential fp32 sum from +0 in list order (torch keeps denormals on the CPU)."""
    assert 1 <= len(srcs) <= 8 and dst.dtype == torch.float32
    acc = torch.zeros(dst.numel(), dtype=torch.float32)
    for s in srcs:
        acc = acc + s.reshape(-1)
    dst.copy_(acc.view(dst.shape))


def install(lib_module):
    """det_ref.install (emu_lib plus the deterministic entry points) plus dp_reduce_det; returns the restore callable."""
    restore_det = det_ref.install(lib_module)
    saved = lib_module.dp_reduce_det
    lib_module.dp_reduce_det = dp_reduce_det

    def restore():
        lib_module.dp_reduce_det = saved
        restore_det()
    return restore
