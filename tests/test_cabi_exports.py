"""The C-ABI library builds for sm_90a without a GPU, loads, and exports every symbol include/qfx.h declares."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_build_and_exports():
    import __graft_entry__ as g
    g.build()
    from qflux_b200.build import LIB
    lib = ctypes.CDLL(LIB)
    hdr = open(os.path.join(ROOT, "include", "qfx.h")).read()
    names = sorted(set(re.findall(r"\b(qfx_[a-z0-9_]+)\s*\(", hdr)))
    assert len(names) >= 18, names
    for n in names:
        assert hasattr(lib, n), f"{n} declared in qfx.h but not exported"
    lib.qfx_last_error.restype = ctypes.c_char_p
    assert lib.qfx_version() >= 1


def test_argument_errors_without_gpu():
    """argument validation happens before any CUDA call, so it is testable on the CPU box."""
    from qflux_b200 import lib
    P = (lib.GemmProblem * 1)()
    rc = lib._lib.qfx_gemm_bf16(P, 1, 128, 100, 0, 0, 1.0, 0, 0, None)
    assert rc != 0 and b"K=100" in lib._lib.qfx_last_error()
