"""qfx_gemm_bf16 per tile and per row (tools/gemm_tile_check.py: each case against an fp64 reference scaled by bf16 eager, the
epilogue's rounding rule on the kernel's own accumulator, sentinels and tests/emu_lib.py), plus the CPU-side checks that need no
GPU: the fp64 references agree with emu_lib, emu_lib refuses what the kernel refuses, and the C ABI refuses bad arguments before
any CUDA call."""
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import gemm_tile_check as gt  # noqa: E402


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(gt.CASES))
def test_gemm_case(name):
    r = gt.CASES[name]()
    print(f"GEMM {name} " + json.dumps(r))
    assert not r["fail"], r["fail"]


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("epi", [gt.EPI_BIAS, gt.EPI_GELU, gt.EPI_RESID_GATE, gt.EPI_DGELU, gt.EPI_ADD, gt.EPI_ATTN_DO])
def test_fp64_gemm_reference_agrees_with_emulation(epi):
    """The references the GPU cases trust, checked on CPU first: the fp64 contraction + epilogue (with a LoRA k-block at
    a2_col0 > 0, three output groups for trans_b = 0) against emu_lib, which rounds like the kernel (so the two differ by bf16
    rounding only, per row); and the rounding rule on emu_lib's own first rounding point reproduces its output."""
    import torch
    import emu_lib as emu
    trans_b = epi in (gt.EPI_BIAS, gt.EPI_DGELU, gt.EPI_ADD, gt.EPI_ATTN_DO) and epi != gt.EPI_BIAS
    M, N, K = 70, 384, 128
    p = gt._prob(M, N, K, trans_b, 1, epi=epi, kb2=2, a2_col0=64, groups=1 if trans_b else 3, bias=not trans_b,
                 rows_per_batch=35 if epi in (gt.EPI_RESID_GATE, gt.EPI_ATTN_DO) else 0, device="cpu")
    alpha = 1.0 if epi in (gt.EPI_GELU, gt.EPI_RESID_GATE) else 0.75
    lgn = 0 if trans_b else 128
    ref = gt.epi_ref(p, gt.acc_ref(p, N, trans_b, lgn), epi, alpha)
    out, out2 = torch.empty(M, N, dtype=torch.bfloat16), torch.empty(M, N, dtype=torch.bfloat16)
    extra = {}
    if epi == gt.EPI_ATTN_DO:
        p.update(rows_per_batch=35, s_offset=2)
        out = torch.zeros(2, N // 128, 40, 128, dtype=torch.bfloat16)
        extra = dict(delta=torch.zeros(2, N // 128, 40), s_offset=2)
    ep = emu.gemm_problem(p["A"], p["B"], out, A2=p["A2"], B2=p["B2"], kb2=2, a2_col0=64, bias=p.get("bias"),
                          out2=out2 if epi in (gt.EPI_GELU, gt.EPI_RESID_GATE, gt.EPI_ATTN_DO) else None, resid=p.get("resid"),
                          gate=p.get("gate"), rows_per_batch=p.get("rows_per_batch", 0), aux=p.get("aux"), **extra)
    emu.gemm([ep], N, K, trans_b=trans_b, epilogue=epi, alpha=alpha, lora_group_n=lgn)
    got = out if epi != gt.EPI_ATTN_DO else out[:, :, 2:37].permute(0, 2, 1, 3).reshape(M, N)
    assert gt.row_rel_max(got, ref["out"]) < 1e-2
    if "out2" in ref:
        assert gt.row_rel_max(out2, ref["out2"]) < 1e-2
    if epi == gt.EPI_ATTN_DO:
        d = extra["delta"][:, :, 2:37].permute(0, 2, 1).reshape(M, -1).double()
        mag = (ref["out"] * p["aux"].double()).abs().view(M, -1, 128).sum(-1)
        assert ((d - ref["delta"]).abs() <= 1e-2 * mag).all()
        assert (out[:, :, :2] == 0).all() and (out[:, :, 37:] == 0).all()
    # a2_col0 matters: the reference without it is far off
    q = dict(p, a2_col0=0)
    assert gt.row_rel_max(got, gt.epi_ref(q, gt.acc_ref(q, N, trans_b, lgn), epi, alpha)["out"]) > 0.1
    if epi not in (gt.EPI_BIAS, gt.EPI_ATTN_DO):  # the rule on emu_lib's own first rounding point
        rb = torch.empty(M, N, dtype=torch.bfloat16)
        emu.gemm([emu.gemm_problem(p["A"], p["B"], rb, A2=p["A2"], B2=p["B2"], kb2=2, a2_col0=64,
                                   bias=p.get("bias") if epi in (gt.EPI_GELU, gt.EPI_RESID_GATE) else None)],
                 N, K, trans_b=trans_b, alpha=1.0 if epi in (gt.EPI_GELU, gt.EPI_RESID_GATE) else alpha, lora_group_n=lgn)
        want = gt.rule(p, rb, epi)["out"]
        if want.dtype == torch.float64:
            assert ((out.double() - want).abs() <= gt._up(want) + 2.0 ** -20 * (1 + want.abs())).all()
        else:
            assert torch.equal(out, want)


def test_emulated_gemm_refuses_alpha_for_gelu_and_resid_gate():
    """qfx.h: alpha scales the accumulator of BIAS / ADD / DGELU / ATTN_DO only; the kernel refuses alpha != 1 for GELU and
    RESID_GATE, and so does the emulation the CPU tests run the model on."""
    import torch
    import emu_lib as emu
    A, W = torch.zeros(4, 64, dtype=torch.bfloat16), torch.zeros(64, 64, dtype=torch.bfloat16)
    o = torch.empty(4, 64, dtype=torch.bfloat16)
    for epi, kw in ((emu.EPI_GELU, dict(out2=torch.empty_like(o))), (emu.EPI_RESID_GATE, dict(resid=o.clone(), gate=torch.ones(1, 64)))):
        with pytest.raises(AssertionError, match="alpha"):
            emu.gemm([emu.gemm_problem(A, W, o, **kw)], 64, 64, epilogue=epi, alpha=0.5)
        emu.gemm([emu.gemm_problem(A, W, o, **kw)], 64, 64, epilogue=epi, alpha=1.0)


def _err(lib):
    return lib._lib.qfx_last_error().decode()


def test_gemm_refuses_bad_arguments_without_gpu():
    """Every problem is validated before any tensor map is encoded, so each refusal below comes back with its message on a machine
    without a driver (a missing check would go on to encode tensor maps and fail differently, or launch on stand-in addresses)."""
    from qflux_b200 import lib
    P = 0x10000  # a 16-byte aligned stand-in address: nothing is dereferenced before the checks
    N, K = 256, 128

    def call(epi, nprob=1, alpha=1.0, trans_b=None, second=None, **kw):
        base = dict(A=P, lda=K, B=P, ldb=K, M=64, out=P, ldo=N, out2=P, ldo2=N, resid=P, ldr=N, gate=P, ldg=N, rows_per_batch=32,
                    aux=P, ldaux=N, delta=P, attn_S=64, attn_H=N // 128)
        tb = epi in (lib.EPI_DGELU, lib.EPI_ADD, lib.EPI_ATTN_DO) if trans_b is None else trans_b
        probs = []
        for i in range(nprob):
            a = dict(base, **(kw if i == nprob - 1 else {}))
            if i == 1 and second:
                a.update(second)
            probs.append(lib.GemmProblem(a["A"], a["lda"], a["B"], a["ldb"], a["M"], a.get("A2", 0), a.get("lda2", 0), a.get("B2", 0),
                                         a.get("ldb2", 0), a.get("kb2", 0), a.get("a2_col0", 0), a.get("bias", 0), a["out"], a["ldo"],
                                         a["out2"], a["ldo2"], a["resid"], a["ldr"], a["gate"], a["ldg"], a["rows_per_batch"], a["aux"],
                                         a["ldaux"], 0, 0, a["delta"] if epi == lib.EPI_ATTN_DO else 0, a["attn_S"], a["attn_H"],
                                         a.get("s_offset", 0)))
        arr = (lib.GemmProblem * nprob)(*probs)
        return lib._lib.qfx_gemm_bf16(arr, nprob, N, K, int(tb), epi, alpha, 0, 128, None)

    refusals = [
        (lambda: call(lib.EPI_GELU, alpha=0.5, out2=P), "alpha = 1 only"),
        (lambda: call(lib.EPI_RESID_GATE, alpha=2.0), "alpha = 1 only"),
        # per-epilogue operands of the LAST problem: these checks used to run after the earlier problems' tensor maps were encoded
        (lambda: call(lib.EPI_GELU, nprob=3, out2=0), "GELU epilogue needs out2"),
        (lambda: call(lib.EPI_RESID_GATE, nprob=2, gate=0), "needs resid+gate"),
        (lambda: call(lib.EPI_ADD, nprob=2, ldr=N + 4), "ADD epilogue needs resid"),
        (lambda: call(lib.EPI_DGELU, nprob=2, aux=0), "DGELU epilogue needs aux"),
        (lambda: call(lib.EPI_ATTN_DO, nprob=2, attn_H=1), "ATTN_DO epilogue needs"),
        (lambda: call(lib.EPI_ATTN_DO, nprob=2, second=dict(attn_S=96)), "must share delta"),
        (lambda: call(lib.EPI_ATTN_DO, s_offset=40), "outside attn_S"),
        (lambda: call(lib.EPI_BIAS, nprob=2, kb2=1, A2=P, B2=0), "bad LoRA operands"),
        (lambda: call(lib.EPI_BIAS, nprob=2, M=0), "null/empty operands"),
        (lambda: call(lib.EPI_BIAS, nprob=2, lda=K + 4), "multiples of 8"),
        # ldo2 of RESID_GATE and ATTN_DO
        (lambda: call(lib.EPI_RESID_GATE, out2=P, ldo2=N + 4), "ldo2"),
        (lambda: call(lib.EPI_ATTN_DO, out2=P, ldo2=N + 2), "ldo2"),
    ]
    # 16-byte bases of every vector-accessed epilogue operand
    for epi, name in ((lib.EPI_BIAS, "out"), (lib.EPI_BIAS, "bias"), (lib.EPI_GELU, "out2"), (lib.EPI_RESID_GATE, "resid"),
                      (lib.EPI_RESID_GATE, "gate"), (lib.EPI_RESID_GATE, "out2"), (lib.EPI_ADD, "resid"), (lib.EPI_DGELU, "aux"),
                      (lib.EPI_ATTN_DO, "aux"), (lib.EPI_ATTN_DO, "out"), (lib.EPI_ATTN_DO, "out2")):
        kw = {name: P + 8}
        if name == "out2" or epi == lib.EPI_GELU:
            kw.setdefault("out2", P)
        refusals.append((lambda epi=epi, kw=kw: call(epi, nprob=2, **kw), "16-byte aligned"))
    for i, (fn, msg) in enumerate(refusals):
        rc = fn()
        assert rc != 0 and msg in _err(lib), (i, msg, _err(lib))
    # a valid call gets past every check and stops only where the driver is needed (or runs, where there is one)
    if not _has_driver():
        rc = call(lib.EPI_RESID_GATE, nprob=2, out2=P)
        assert rc != 0 and "cuTensorMapEncodeTiled" in _err(lib), _err(lib)


def _has_driver():
    import torch
    return torch.cuda.is_available()
