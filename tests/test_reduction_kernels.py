"""The backward's fp32 reductions (LoRA weight gradients on the tensor cores and on CUDA cores, the modulation gradients, the
flow-matching loss) and the conditioning GEMV, per element against fp64 at their split and tile edges (tools/reduce_check.py, with
sentinels around every output and the `_det` twins under the same bound), plus the CPU-side checks that need no GPU: the fp64
reference helpers agree with tests/emu_lib.py, the restated split plans agree with the C side's scratch rules, and the C ABI refuses
the arguments that would crash these kernels before any CUDA call."""
import json
import os
import subprocess
import sys
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import reduce_check as rc  # noqa: E402


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(rc.CASES))
def test_reduction_case(name):
    r = rc.CASES[name]()
    print(f"REDUCE {name} " + json.dumps(r))
    assert not r["fail"], r["fail"][:20]


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_fp64_references_agree_with_emulation():
    """The references the GPU cases trust, checked against emu_lib (fp32 torch on the CPU) at small shapes: the reductions within the
    fp32 reduction bound, the GEMV within its rounding bound, and dpred bit for bit against the stated fp32 rule."""
    import torch
    import emu_lib as emu
    BF = torch.bfloat16

    def close(got, ref, mag):
        assert ((got.double() - ref).abs() <= rc.RED_TOL * mag + 1e-30).all()
    # wgrad_tc, both modes, the dA store of emu_lib's strided view
    M, Na, G, r = 77, 256, 3, 7
    B = rc._mk(M, 64 * G, seed=2, device="cpu")
    for mode, Dg, na in ((0, 0, Na), (1, 128, 3 * 128)):
        A = rc._mk(M, na, seed=3, device="cpu")
        rows = Dg if mode else na
        Gs = [torch.zeros(rows * r) for _ in range(G)]
        emu.lora_wgrad_tc(A, B, Gs, 1, rows, r, mode=mode, Dg=Dg)
        for g, (ref, mag) in enumerate(rc.wgrad_tc_ref(A, B, r, G, mode, Dg)):
            close(torch.as_strided(Gs[g], (rows, r), (1, rows)), ref, mag)
    # lora_wgrad with a column-sliced Q
    P, Qb = rc._mk(70, 100, seed=4, device="cpu"), rc._mk(70, 192, seed=5, device="cpu")
    Q = Qb[:, 64:80]
    Gl = torch.zeros(100 * 16)
    emu.lora_wgrad(P, Q, Gl, 16, 1, 16)
    ref, mag = rc.lora_wgrad_ref(P, Q, 16)
    close(Gl.view(100, 16), ref, mag)
    # mod_grad, the three forms
    rpb, D = 33, 24
    g, m = rc._mk(3 * rpb, D, seed=6, device="cpu"), rc._mk(3 * rpb, D, seed=7, scale=2.0, shift=0.5, device="cpu")
    mean, rstd = m.float().mean(1), torch.rsqrt(m.float().var(1, unbiased=False) + 1e-6)
    for mm, mu, rs in ((None, None, None), (m, mean, rstd), (m, None, None)):
        so, po = torch.zeros(3, D), torch.zeros(3, D)
        emu.mod_grad(g, rpb, sum_out=so, m=mm, prod_out=po if mm is not None else None, mean=mu, rstd=rs)
        ref = rc.mod_grad_ref(g, rpb, mm, mu, rs)
        close(so, ref["sum"], ref["sum_mag"])
        if mm is not None:
            assert ((po.double() - ref["prod"]).abs() <= rc.RED_TOL * ref["prod_mag"] + ref["flip"] + 1e-30).all()
    # flow_loss: the fp32 dpred rule is emu_lib's expression, bit for bit; loss within the reduction bound
    Bn, L, Ltot, C = 2, 9, 12, 16
    x0, nz, pred = (rc._mk(Bn, n, C, seed=s, device="cpu") for s, n in ((8, L), (9, L), (10, Ltot)))
    w = torch.rand(Bn, L, generator=torch.Generator().manual_seed(0)) + 0.5
    for ww in (None, w):
        for gs in (1.0, 0.25):
            loss, dp = torch.zeros(1), torch.empty(Bn, Ltot, C, dtype=BF)
            emu.flow_loss(pred, x0, nz, ww, 1.0 / (Bn * L * C), loss, dp, gs)
            l64, lmag, rule, dp64 = rc.flow_loss_ref(pred, x0, nz, ww, 1.0 / (Bn * L * C), gs)
            assert torch.equal(dp.view(torch.int16), rule.view(torch.int16))
            assert ((dp.double() - dp64).abs() <= rc._up(dp64)).all()
            assert abs(loss.double().item() - l64.item()) <= rc.RED_TOL * lmag.item()
    # gemv_act, both activations, with and without bias
    x, W, bias = rc._mk(3, 64, seed=11, scale=2.0, device="cpu"), rc._mk(10, 64, seed=12, scale=0.125, device="cpu"), rc._mk(10, seed=13, device="cpu")
    for act in (0, 1):
        for b in (None, bias):
            y = torch.empty(3, 10, dtype=BF)
            emu.gemv_act(x, W, b, y, act)
            ref, mag, flip = rc.gemv_ref(x, W, b, act)
            assert ((y.double() - ref).abs() <= rc.RED_TOL * mag + flip + rc._up(torch.maximum(y.double().abs(), ref.abs()))).all()


def test_split_plans_restate_the_host_formulas():
    """With 132 SMs the atomic kernels' split counts equal the deterministic twins' fixed ones (2 x 132 = QFX_DET_WGRAD_CTAS,
    4 x 132 = QFX_DET_MODGRAD_CTAS), so the restated plans must reproduce lib.det_scratch_*; and every edge the GPU cases derive has
    the property it is named after."""
    from qflux_b200 import lib
    for Na in (128, 384, 3072, 12288):
        for M in (1, 63, 64, 65, 256, 257, 769, 1408, 3000, 8192):
            p = rc.wgrad_tc_plan(M, Na, 132)
            assert p["grid_splits"] * Na * 2 * 16 == lib.det_scratch_wgrad_tc(M, Na, 2, 16), (M, Na)
            assert 1 <= p["last"] <= p["rows"] and p["rows"] % 64 == 0
    for B in (1, 3, 8):
        for D in (8, 264, 3072):
            for rpb in (1, 31, 32, 33, 352, 1025, 4097):
                p = rc.mod_grad_plan(rpb, B, D, 132)
                assert p["splits"] * 2 * B * D == lib.det_scratch_mod_grad(B * rpb, rpb, D), (B, D, rpb)
                assert p["grid_splits"] == p["splits"]  # no empty split at these shapes
    for sms in (114, 132):
        for Na in (128, 3072):
            plan = lambda M: rc.wgrad_tc_plan(M, Na, sms)  # noqa: E731
            e = rc.split_edges(plan, 257, 1 << 18, 64)
            assert all(plan(v)["sm_bound"] for v in e.values())
            assert plan(e["last_one_row"])["last"] == 1 and plan(e["last_one_kblock"])["last"] == 64 and e["mult64"] % 64 == 0
            exact = plan(e["fill_minus1"] + 1)
            assert exact["rows"] * exact["grid_splits"] == e["fill_minus1"] + 1 == e["fill_plus1"] - 1
        for B, D in ((1, 3072), (3, 264), (8, 3072)):
            plan = lambda v: rc.mod_grad_plan(v, B, D, sms)  # noqa: E731
            e = rc.split_edges(plan, 33, 1 << 15, 8)
            assert all(plan(v)["sm_bound"] and plan(v)["grid_splits"] >= 2 for v in e.values())
            assert e["mult64"] % 64 == 0 and plan(e["fill_minus1"] + 1)["rows"] * plan(e["fill_minus1"] + 1)["grid_splits"] == e["fill_minus1"] + 1
            if B * D < 8 * 3072:  # enough SM-set splits for these two edges (split_edges' docstring)
                assert plan(e["last_one_row"])["last"] == 1 and plan(e["last_one_kblock"])["last"] == 8


def _err(lib):
    return lib._lib.qfx_last_error().decode()


def test_reduction_entry_points_refuse_bad_arguments_without_gpu():
    """Argument validation happens before any CUDA call: a rank the CUDA-core wgrad has no kernel for, null or misaligned operands,
    leading dimensions the 16-byte accesses cannot use and an inconsistent loss shape are refused with a message, never launched."""
    from qflux_b200 import lib
    P = 0x10000  # a 16-byte aligned stand-in address: nothing is dereferenced before the checks
    M, D, rpb = 64, 512, 32

    def mod_grad(g=P, ldg=D, m=P, ldm=D, M=M, D=D, rpb=rpb, det=False):
        if det:
            return lib._mod_grad_det(g, ldg, m, ldm, None, None, rpb, P, P, 6 * D, M, D, P, 1 << 30, None)
        return lib._mod_grad(g, ldg, m, ldm, None, None, rpb, P, P, 6 * D, M, D, None)

    def gate_mul(a=P, lda=D, gate=P, ldg=3 * D, out=P, ldo=D):
        return lib._gate_mul(a, lda, gate, ldg, rpb, out, ldo, M, D, None)

    def flow_loss(loss=P, B=2, L=16, Ltot=16, C=64):
        return lib._floss(P, P, P, None, 1.0, 1.0, loss, P, B, L, Ltot, C, None)

    def wgrad(G=P, r=16, M=M, Dp=64):
        return lib._wgrad(P, 64, P, 192, G, r, 1, M, Dp, r, None)

    refusals = [(lambda: wgrad(r=12), "rank 12 unsupported"), (lambda: wgrad(G=None), "qfx_lora_wgrad: bad arguments"),
                (lambda: wgrad(Dp=0), "qfx_lora_wgrad: bad arguments"), (lambda: wgrad(M=-1), "qfx_lora_wgrad: bad arguments"),
                (lambda: flow_loss(Ltot=15), "qfx_flow_loss: bad arguments"), (lambda: flow_loss(loss=None), "qfx_flow_loss: bad arguments"),
                (lambda: flow_loss(B=0), "qfx_flow_loss: bad arguments"), (lambda: flow_loss(L=0, Ltot=0), "qfx_flow_loss: bad arguments"),
                (lambda: flow_loss(C=0), "qfx_flow_loss: bad arguments")]
    for det in (False, True):
        name = "qfx_mod_grad_det" if det else "qfx_mod_grad"
        refusals += [(lambda det=det: mod_grad(g=P + 8, det=det), f"{name}: g / m must be 16-byte aligned"),
                     (lambda det=det: mod_grad(m=P + 8, det=det), f"{name}: g / m must be 16-byte aligned"),
                     (lambda det=det: mod_grad(D=-8, det=det), f"{name}: bad dims"),
                     (lambda det=det: mod_grad(M=-32, det=det), f"{name}: bad dims")]
    for kw in (dict(a=P + 8), dict(gate=P + 8), dict(out=P + 2)):
        refusals.append((lambda kw=kw: gate_mul(**kw), "qfx_gate_mul: operands must be 16-byte aligned"))
    for kw in (dict(lda=D + 4), dict(ldg=3 * D + 2), dict(ldo=D + 1)):
        refusals.append((lambda kw=kw: gate_mul(**kw), "qfx_gate_mul: leading dimensions must be multiples of 8"))
    for i, (call, msg) in enumerate(refusals):
        r = call()
        assert r != 0 and msg in _err(lib), (i, msg, _err(lib))


def test_zero_rows_and_zero_width_are_refused_in_a_subprocess():
    """M = 0 and D = 0 reach a division by the split count in qfx_lora_wgrad / qfx_mod_grad(_det) unless they are refused first.  The
    calls run in a child process, so a division fault shows up as this test failing rather than as a dead pytest run."""
    script = textwrap.dedent(f"""
        import sys
        sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, "qwen-image-finetune_b200")!r}]
        from qflux_b200 import lib
        P = 0x10000
        calls = [
            ("lora_wgrad M=0", lambda: lib._wgrad(P, 64, P, 192, P, 16, 1, 0, 64, 16, None), "qfx_lora_wgrad: bad arguments"),
            ("mod_grad M=0", lambda: lib._mod_grad(P, 512, P, 512, None, None, 32, P, P, 3072, 0, 512, None), "qfx_mod_grad: bad dims"),
            ("mod_grad D=0", lambda: lib._mod_grad(P, 512, P, 512, None, None, 32, P, P, 3072, 64, 0, None), "qfx_mod_grad: bad dims"),
            ("mod_grad_det M=0", lambda: lib._mod_grad_det(P, 512, P, 512, None, None, 32, P, P, 3072, 0, 512, P, 1 << 30, None),
             "qfx_mod_grad_det: bad dims"),
            ("mod_grad_det D=0", lambda: lib._mod_grad_det(P, 512, P, 512, None, None, 32, P, P, 3072, 64, 0, P, 1 << 30, None),
             "qfx_mod_grad_det: bad dims"),
        ]
        for name, call, msg in calls:
            rc = call()
            print(name, "|", rc, "|", msg in lib._lib.qfx_last_error().decode(), "|", lib._lib.qfx_last_error().decode(), flush=True)
    """)
    r = subprocess.run([sys.executable, "-c", script], capture_output=True, text=True, timeout=300, cwd=ROOT)
    assert r.returncode == 0, f"child died with {r.returncode}:\n{r.stdout}\n{r.stderr[-2000:]}"
    lines = [ln.split(" | ") for ln in r.stdout.splitlines() if " | " in ln]
    assert len(lines) == 5, r.stdout
    for name, code, ok, msg in lines:
        assert code != "0" and ok == "True", (name, code, msg)
