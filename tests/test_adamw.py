"""The optimizer tail of a training step: clip + AdamW (qfx.h qfx_fused_adamw / FusedLoraAdamW) and clip + bf16 gradient
(qfx_grad_finalize / finalize_grads), against tests/adamw_ref.py, the fp64 restatement of clip_grad_norm_ + torch.optim.AdamW.

CPU: the restatement against torch.optim.AdamW and clip_grad_norm_ on fp64 tensors under a cosine warm-up schedule; tests/emu_lib.py's
fused_adamw against it; the power of the per-element bounds (every listed kernel mistake, run in fp32 through tools/adamw_check.py's
hyper-parameter grid, fails the bounds the GPU case applies); the C entry points' argument refusals, which need no driver.
GPU (tools/adamw_check.py, one subprocess per case): every adamw_check.CASES entry."""
import ctypes as C
import json
import os
import subprocess
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tools"))
CHECK = os.path.join(ROOT, "tools", "adamw_check.py")

import adamw_ref as ar  # noqa: E402
import adamw_check as ac  # noqa: E402


def _problem(shapes, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(s, generator=g, dtype=torch.float64) * 2 for s in shapes]


@pytest.mark.parametrize("max_norm", [0.0, 1.0, 1e3])
@pytest.mark.parametrize("betas", [(0.9, 0.999), (0.0, 0.99), (0.9, 0.9999)])
def test_restatement_matches_torch_adamw_and_clip_grad_norm(betas, max_norm):
    """adamw_ref (torch mode) against torch.optim.AdamW + clip_grad_norm_ on fp64 tensors: 8 steps of a cosine warm-up schedule with
    weight decay, the clip above / below / off; parameters, moments and the norm agree to ~1e-12."""
    shapes = [(7, 5), (3,), (4, 4)]
    ps = [torch.nn.Parameter(t.clone()) for t in _problem(shapes, 1)]
    opt = torch.optim.AdamW(ps, lr=3e-2, betas=betas, eps=1e-3, weight_decay=0.1)
    sch = ar.cosine_warmup(opt, 3, 8)
    mine = [t.clone() for t in _problem(shapes, 1)]
    m = [torch.zeros_like(t) for t in mine]
    v = [torch.zeros_like(t) for t in mine]
    for step in range(1, 9):
        gs = _problem(shapes, 100 + step)
        lr = opt.param_groups[0]["lr"]
        for p, g in zip(ps, gs):
            p.grad = g.clone()
        norm = torch.nn.utils.clip_grad_norm_(ps, max_norm) if max_norm > 0 else None
        opt.step()
        sch.step()
        flat = lambda ts: torch.cat([t.reshape(-1) for t in ts])
        S = ar.scalars("torch", lr, betas[0], betas[1], 1e-3, 0.1, step, 1.0, max_norm)
        R = ar.step_ref(flat(mine), flat(gs), flat(m), flat(v), S)
        if norm is not None:
            assert abs(R["sumsq"] ** 0.5 - float(norm)) <= 1e-12 * float(norm)
        off = 0
        for i, t in enumerate(mine):
            sl = slice(off, off + t.numel())
            mine[i], m[i], v[i] = R["p"][sl].view(t.shape), R["m"][sl].view(t.shape), R["v"][sl].view(t.shape)
            off += t.numel()
        for p, q, a, b in zip(ps, mine, m, v):
            st = opt.state[p]
            assert torch.allclose(p.detach(), q, rtol=1e-12, atol=1e-14)
            assert torch.allclose(st["exp_avg"], a, rtol=1e-12, atol=1e-300)
            assert torch.allclose(st["exp_avg_sq"], b, rtol=1e-12, atol=1e-300)


def test_abi_scalars_differ_from_torch_as_stated():
    """The two modes' sqrt(bc2): 6e-6 relative at beta2 = 0.999, up to ~1.1e-4 at 0.9999; TORCH_P_REL covers the latter."""
    gap = lambda b2, s: abs(ar.scalars("abi", 1, 0, b2, 0, 0, s)["bc2_sqrt"] / ar.scalars("torch", 1, 0, b2, 0, 0, s)["bc2_sqrt"] - 1)
    assert max(gap(0.999, s) for s in (1, 2, 3, 999)) < 1e-5
    g9999 = max(gap(0.9999, s) for s in (1, 2, 3, 999))
    assert 5e-5 < g9999 < ar.TORCH_P_REL


def test_emulated_fused_adamw_agrees_with_the_abi_restatement():
    """tests/emu_lib.py's fused_adamw (what the CPU suite trains with) passes the GPU case's per-element bounds in both modes, at
    every beta, decay and clip of the grid."""
    import emu_lib
    sumsq = torch.zeros(1)

    def step_fn(p, g, m, v, hp, step):
        buf = p.view(-1, 64)
        emu_lib.fused_adamw(([(buf, 0)], None), g, m, v, sumsq, hp["pre_scale"], hp["max_norm"], hp["lr"], hp["beta1"], hp["beta2"],
                            hp["eps"], hp["weight_decay"], step)
        return float(sumsq)
    pts = [pt for pt in ac.grid() if pt[1]["lr"] == 1e-2 and pt[1]["eps"] == 1e-8 and pt[1]["pre_scale"] == 1.0]
    stats, fail = ac.run_grid(step_fn, 1024, "cpu", points=pts)
    assert not fail, fail[:5]


def _fp32_step_fn(mutation):
    def step_fn(p, g, m, v, hp, step):
        gs = g * torch.tensor(ar.scalars("abi", 1, 0, 0, 0, 0, 1, hp["pre_scale"])["pre_scale"], dtype=torch.float32)
        ss = float((gs * gs).sum())
        p.copy_(ar.kernel_fp32(p, g, m, v, hp, step, ss, mutation))
        return ss
    return step_fn


def test_fp32_kernel_arithmetic_passes_the_whole_grid():
    """fused_adamw_kernel's arithmetic, run in fp32 on the CPU, passes every hyper_grid point in both modes with the GPU case's
    bounds: the bounds hold for a correct kernel."""
    stats, fail = ac.run_grid(_fp32_step_fn("none"), 512, "cpu")
    assert not fail, fail[:5]
    assert stats["points"] == len(ac.grid()) == 4 * 2 * 3 * 2 * 2 * 3 + 1


@pytest.mark.parametrize("mutation", [m for m in ar.MUTATIONS if m != "none"])
def test_every_listed_kernel_mistake_fails_the_gpu_bounds(mutation):
    """Power check: the kernel's fp32 arithmetic with one mistake (weight decay dropped, bias correction dropped, the step count off
    by one, eps inside the sqrt, bc2 without its sqrt, the clip ignored) fails the per-element bounds of the GPU case at one of its
    grid points.  Also reports where, so a loosened bound shows up here first."""
    stats, fail = ac.run_grid(_fp32_step_fn(mutation), 512, "cpu", modes=("abi",), stop_at_first_failure=True)
    assert fail, f"{mutation} passes every grid point"
    print(mutation, stats.get("first_failure"), fail[0])


def test_weight_decay_and_bias_correction_slips_fail_at_the_configs_defaults():
    """At torch.optim.AdamW's defaults with parameters of magnitude 1-4 and lr 1e-2, dropping the decay or the bias correction is
    caught on its own (not only somewhere in the grid)."""
    pt = [p for p in ac.grid() if p[0] == "b0.9_0.999_eps1e-08_wd0.5_lr0.01_ps1.0_clipoff"]
    for mut in ("no_weight_decay", "no_bias_correction", "step_off_by_one", "eps_inside_sqrt", "bc2_without_sqrt"):
        _, fail = ac.run_grid(_fp32_step_fn(mut), 512, "cpu", modes=("abi",), points=pt)
        assert fail, mut


def test_c_entry_points_refuse_bad_arguments_before_any_cuda_call():
    """qfx_fused_adamw, qfx_grad_finalize and their _det variants: step < 1, no chunks, an empty gradient, null pointers and a short
    scratch come back as errors with a message; nothing is launched (the machine may have no driver)."""
    from qflux_b200 import lib
    L = lib._lib
    buf = torch.zeros(4096, dtype=torch.float32)
    P = buf.data_ptr()
    vp = C.c_void_p
    f = C.c_float
    for name in ("qfx_fused_adamw", "qfx_fused_adamw_det", "qfx_grad_finalize", "qfx_grad_finalize_det"):
        getattr(L, name).restype = C.c_int

    def adamw(det=False, tensors=P, chunks=P, n_chunks=1, grad=P, n_grad=100, m=P, v=P, sumsq=P, step=1, scratch=P,
              scratch_floats=lib.DET_NORM_PARTIALS):
        a = [vp(tensors), vp(chunks), n_chunks, vp(grad), C.c_int64(n_grad), vp(m), vp(v), vp(sumsq), f(1.0), f(1.0), f(1e-3), f(0.9),
             f(0.999), f(1e-8), f(0.0), step]
        if det:
            return L.qfx_fused_adamw_det(*a, vp(scratch), C.c_int64(scratch_floats), None)
        return L.qfx_fused_adamw(*a, None)

    def gfin(det=False, g=P, n=100, sumsq=P, out=P, scratch=P, scratch_floats=lib.DET_NORM_PARTIALS):
        a = [vp(g), C.c_int64(n), f(1.0), f(1.0), vp(sumsq), vp(out)]
        if det:
            return L.qfx_grad_finalize_det(*a, vp(scratch), C.c_int64(scratch_floats), None)
        return L.qfx_grad_finalize(*a, None)

    cases = []
    for det in (False, True):
        name = "qfx_fused_adamw_det" if det else "qfx_fused_adamw"
        for bad in (dict(step=0), dict(step=-3), dict(n_chunks=0), dict(n_grad=0), dict(tensors=0), dict(chunks=0), dict(grad=0),
                    dict(m=0), dict(v=0), dict(sumsq=0)):
            cases.append((lambda det=det, bad=bad: adamw(det, **bad), f"{name}: bad arguments"))
        name = "qfx_grad_finalize_det" if det else "qfx_grad_finalize"
        for bad in (dict(n=0), dict(n=-1), dict(g=0), dict(sumsq=0), dict(out=0)):
            cases.append((lambda det=det, bad=bad: gfin(det, **bad), f"{name}: bad arguments"))
    cases += [(lambda: adamw(True, scratch_floats=lib.DET_NORM_PARTIALS - 1), "needs 592"), (lambda: adamw(True, scratch=0), "needs 592"),
              (lambda: gfin(True, scratch_floats=lib.DET_NORM_PARTIALS - 1), "needs 592"), (lambda: gfin(True, scratch=0), "needs 592")]
    for i, (fn, msg) in enumerate(cases):
        rc = fn()
        err = L.qfx_last_error().decode()
        assert rc == -1 and msg in err, (i, rc, err)


# ---------------------------------------------------------------------------------------------------- GPU
def _run_case(name):
    r = subprocess.run([sys.executable, CHECK, "--case", name], capture_output=True, text=True, timeout=1500, cwd=ROOT)
    res = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
    assert r.returncode == 0 and res, (r.stdout + r.stderr)[-3000:]
    out = json.loads(res[-1][7:])
    print(name, json.dumps(out))
    assert not out.get("fail"), out
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(ac.CASES))
def test_adamw_on_gpu(case):
    _run_case(case)
