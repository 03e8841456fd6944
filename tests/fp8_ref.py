"""TEST INFRASTRUCTURE ONLY — the FP8 side of the FP8 tests in plain PyTorch:

  * `fp8_expand` emulates the `qflux_b200.lib.fp8_expand` entry point for `-m "not gpu"` runs: torch's e4m3fn -> bf16 conversion,
    which tools/fp8_check.py holds the kernel to bit for bit on every code (see emu_lib.py for the other entry points).
"""
from __future__ import annotations

import torch

import emu_lib


def fp8_expand(segments):
    for codes, out in segments:
        out.copy_(codes.reshape(-1).view(torch.float8_e4m3fn).to(torch.bfloat16).view(out.shape))


def install(lib_module):
    """emu_lib.install plus the FP8 entry point; returns the restore callable."""
    restore_emu = emu_lib.install(lib_module)
    saved = lib_module.fp8_expand
    lib_module.fp8_expand = fp8_expand

    def restore():
        lib_module.fp8_expand = saved
        restore_emu()
    return restore
