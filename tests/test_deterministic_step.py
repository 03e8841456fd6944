"""Bit-reproducible training steps under torch.use_deterministic_algorithms(True).

CPU: with tests/emu_lib.py and tests/det_ref.py in place of the kernels, the flag switches every reduction of the step to its
deterministic entry point (and nothing else), the workspace gains the reduction scratch sized by qfx.h's rules, flag-off steps call exactly what they called
before, the CUDA-graph key separates the two settings, and every new C entry point refuses bad arguments before any CUDA call.
GPU (tools/determinism_check.py, one subprocess per case, each with the flag on and CUBLAS_WORKSPACE_CONFIG set): the kernels
against fp64 bounds and across launches, two processes giving the same SHA-256 digests for three optimizer steps, the equalities
that now hold bit for bit, and tools/lora_grad_check.py's per-tensor accuracy on the deterministic path."""
import ctypes as C
import json
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
CHECK = os.path.join(ROOT, "tools", "determinism_check.py")

DET_NAMES = ("attn_bwd_det", "lora_wgrad_tc_det", "lora_wgrad_det", "mod_grad_det", "flow_loss_det", "grad_finalize_det",
             "fused_adamw_det")
ATOMIC_NAMES = ("attn_bwd", "lora_wgrad_tc", "lora_wgrad", "mod_grad", "flow_loss", "grad_finalize", "fused_adamw")


@pytest.fixture()
def emu():
    import det_ref
    from qflux_b200 import lib
    restore = det_ref.install(lib)
    yield lib
    restore()


@pytest.fixture()
def deterministic():
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(was)


def _traced(lib, names):
    """wrap lib.<name> for every name; returns the call log [(name, n_positional, sorted keywords)]"""
    log = []
    for n in names:
        f = getattr(lib, n)

        def w(*a, _f=f, _n=n, **k):
            log.append((_n, len(a), tuple(sorted(k))))
            return _f(*a, **k)
        setattr(lib, n, w)
    return log


def _qwen_step(lib, targets=("to_q", "to_v", "to_out.0", "img_mlp.net.2", "img_mod.1", "txt_mod.1", "img_in", "txt_in")):
    import lora_grad_check as lg
    from qflux_b200.optim import FusedLoraAdamW
    from qflux_b200.train_step import QwenImageEditStep
    orc, m = lg.qwen_pair(torch.device("cpu"), targets=targets)
    g = torch.Generator().manual_seed(0)
    B, hw, T = 2, 4, 24
    rn = lambda *s: torch.randn(*s, generator=g).bfloat16()
    emb = dict(image_latents=rn(B, hw * hw, 64), control_latents=rn(B, hw * hw, 64), prompt_embeds=rn(B, T, m.J) * 3,
               img_shapes=[[(1, hw, hw), (1, hw, hw)]] * B)
    step = QwenImageEditStep(m, use_cuda_graph=False)
    opt = FusedLoraAdamW(m, lr=1e-3)
    return m, step, opt, emb, rn(B, hw * hw, 64)


def _run_steps(lib, n=2):
    m, step, opt, emb, noise = _qwen_step(lib)
    losses = [float(step.train_step(emb, opt, noise=noise, u=torch.tensor([0.5, 0.25]))) for _ in range(n)]
    m.finalize_grads(1, 1.0)
    return m, losses


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_flag_selects_the_deterministic_entry_points(emu, deterministic):
    log = _traced(emu, DET_NAMES + ATOMIC_NAMES)
    m, losses = _run_steps(emu)
    called = {n for n, _, _ in log}
    assert called == set(DET_NAMES), called
    assert m._ws["det"] and m._ws["det_scratch"].numel() == m._det_scratch_floats(m._ws["B"], m._ws["T"], m._ws["Limg"])
    assert m._ws_key[3:] == (True, True)
    assert all(l == l for l in losses)


def test_flag_off_calls_what_it_called_before(emu):
    """No deterministic entry point, no scratch; the call sequence of the atomic entry points is the same with the flag off as with
    the flag on, entry point for entry point (only the names and the scratch keyword differ)."""
    assert not torch.are_deterministic_algorithms_enabled()
    log = _traced(emu, DET_NAMES + ATOMIC_NAMES)
    m, off = _run_steps(emu)
    assert {n for n, _, _ in log} == set(ATOMIC_NAMES) and not m._ws["det"] and "det_scratch" not in m._ws
    seq_off = [(n, a, k) for n, a, k in log]
    log.clear()
    torch.use_deterministic_algorithms(True)
    try:
        _, on = _run_steps(emu)
    finally:
        torch.use_deterministic_algorithms(False)
    seq_on = [(n[:-4], a, tuple(x for x in k if x != "scratch")) for n, a, k in log]
    assert seq_on == seq_off
    assert on == off  # the emulation computes the same either way


def test_workspace_counts_the_scratch_only_under_the_flag(emu):
    from qflux_b200 import lib
    m, step, opt, emb, noise = _qwen_step(emu)
    B, T, Limg = 2, 24, 32
    _, post_off = m._fixed_entries(B, T, Limg, True, m.L, (), False)
    _, post_on = m._fixed_entries(B, T, Limg, True, m.L, (), True)
    extra = [e for e in post_on if e not in post_off]
    assert [e[0] for e in extra] == ["det_scratch"] and extra[0][2] == torch.float32
    assert extra[0][1][0] >= max(lib.DET_LOSS_PARTIALS, lib.det_scratch_mod_grad(B * Limg, Limg, m.D))
    _, post_inf = m._fixed_entries(B, T, Limg, False, m.L, (), True)
    assert "det_scratch" not in [e[0] for e in post_inf]


def test_scratch_rules_match_the_kernel_grids():
    from qflux_b200 import lib
    # wgrad_tc: Na = 3072 -> 24 tiles -> at most 11 splits; M = 4096 -> 11 splits of 384 rows
    assert lib.det_scratch_wgrad_tc(4096, 3072, 3, 16) == 11 * 3072 * 3 * 16
    assert lib.det_scratch_wgrad_tc(100, 3072, 1, 16) == 1 * 3072 * 16
    assert lib.det_scratch_wgrad(2048, 64, 16) == 4 * 64 * 16
    assert lib.det_scratch_mod_grad(2 * 1024, 1024, 3072) == 22 * 2 * 2 * 3072  # ceil(528 / 24) = 22 <= ceil(1024 / 32)


def test_graph_key_separates_the_two_settings():
    from qflux_b200.mmdit_base import GraphCache

    class M:
        _sharded, dev = None, torch.device("cuda")
    cache = GraphCache(4, "test")
    real = torch.cuda.is_available
    torch.cuda.is_available = lambda: True
    try:
        cache.run(M(), lambda x: x, (1,), tag=False)
        torch.use_deterministic_algorithms(True)
        try:
            cache.run(M(), lambda x: x, (1,), tag=False)
        finally:
            torch.use_deterministic_algorithms(False)
    finally:
        torch.cuda.is_available = real
    keys = list(cache.entries)
    assert len(keys) == 2 and keys[0][:2] == keys[1][:2] and keys[0][2] != keys[1][2]


def test_deterministic_entry_points_refuse_bad_arguments_without_gpu():
    """Each refusal comes back with its message before any CUDA call (the machine may have no driver)."""
    from qflux_b200 import lib
    L = lib._lib
    buf = torch.zeros(1 << 16, dtype=torch.float32)
    p = buf.data_ptr() + (-buf.data_ptr()) % 16
    vp = C.c_void_p
    G = (C.c_void_p * 3)(p, p, p)
    stream = vp(0)
    refusals = [
        (lambda: L.qfx_attn_bwd_det(vp(p), vp(p), vp(p), vp(p), vp(p), vp(p), vp(p), vp(p), vp(p), None, None, 0, 0, 1, 128, 0.1, stream),
         "qfx_attn_bwd_det: bad arguments"),
        (lambda: L.qfx_attn_bwd_det(vp(p), vp(p), vp(p), vp(p), vp(p), vp(p), vp(p), vp(p), vp(p), None, vp(p), 0, 1, 1, 128, 0.1, stream),
         "txt_len needs 0 < split <= S"),
        (lambda: L.qfx_attn_bwd_det(vp(p), vp(p), vp(p), vp(p), vp(p), vp(p), vp(p + 4), vp(p), vp(p), None, None, 0, 1, 1, 128, 0.1,
                                    stream), "dQ_accum must be 8-byte aligned"),
        (lambda: L.qfx_lora_wgrad_tc_det(vp(p), 256, 100, vp(p), 64, 1, 512, 0, 0, G, 16, 1, 16, vp(p), 1 << 20, stream), "bad shape"),
        (lambda: L.qfx_lora_wgrad_tc_det(vp(p), 256, 256, vp(p), 64, 2, 512, 1, 64, G, 16, 1, 16, vp(p), 1 << 20, stream), "bad mode/Dg"),
        (lambda: L.qfx_lora_wgrad_tc_det(vp(p), 250, 256, vp(p), 64, 1, 512, 0, 0, G, 16, 1, 16, vp(p), 1 << 20, stream),
         "multiples of 8"),
        (lambda: L.qfx_lora_wgrad_tc_det(vp(p), 256, 256, vp(p), 64, 1, 512, 0, 0, G, 16, 1, 16, vp(p), 256 * 16 * 2 - 1, stream),
         "needs 8192"),
        (lambda: L.qfx_lora_wgrad_tc_det(vp(p), 256, 256, vp(p), 64, 1, 512, 0, 0, G, 16, 1, 16, None, 1 << 20, stream), "needs"),
        (lambda: L.qfx_lora_wgrad_det(vp(p), 64, vp(p), 64, vp(p), 1, 64, 512, 64, 12, vp(p), 1 << 20, stream), "rank 12 unsupported"),
        (lambda: L.qfx_lora_wgrad_det(vp(p), 64, vp(p), 64, vp(p), 1, 64, 1024, 64, 16, vp(p), 2 * 64 * 16 - 1, stream), "needs 2048"),
        (lambda: L.qfx_mod_grad_det(vp(p), 256, None, 0, None, None, 100, vp(p), None, 256, 250, 256, vp(p), 1 << 20, stream), "bad dims"),
        (lambda: L.qfx_mod_grad_det(vp(p), 256, None, 0, vp(p), vp(p), 100, vp(p), None, 256, 200, 256, vp(p), 1 << 20, stream),
         "mean/rstd need m"),
        (lambda: L.qfx_mod_grad_det(vp(p), 256, None, 0, None, None, 64, vp(p), None, 256, 128, 256, vp(p), 2 * 2 * 2 * 256 - 1, stream),
         "needs 2048"),
        (lambda: L.qfx_flow_loss_det(vp(p), vp(p), vp(p), None, C.c_float(1.0), C.c_float(1.0), vp(p), None, 1, 16, 32, 64, vp(p), 295,
                                     stream), "needs 296"),
        (lambda: L.qfx_flow_loss_det(vp(p), vp(p), vp(p), None, C.c_float(1.0), C.c_float(1.0), None, None, 1, 16, 32, 64, vp(p), 296,
                                     stream), "bad arguments"),
        (lambda: L.qfx_grad_finalize_det(vp(p), 100, C.c_float(1.0), C.c_float(1.0), vp(p), vp(p), vp(p), 591, stream), "needs 592"),
        (lambda: L.qfx_grad_finalize_det(vp(p), 0, C.c_float(1.0), C.c_float(1.0), vp(p), vp(p), vp(p), 592, stream), "bad arguments"),
        (lambda: L.qfx_fused_adamw_det(vp(p), vp(p), 1, vp(p), 100, vp(p), vp(p), vp(p), *[C.c_float(1.0)] * 7, 1, vp(p), 591, stream),
         "needs 592"),
        (lambda: L.qfx_fused_adamw_det(vp(p), vp(p), 1, vp(p), 100, vp(p), vp(p), vp(p), *[C.c_float(1.0)] * 7, 0, vp(p), 592, stream),
         "bad arguments"),
    ]
    for fn_name in ("qfx_attn_bwd_det", "qfx_lora_wgrad_tc_det", "qfx_lora_wgrad_det", "qfx_mod_grad_det", "qfx_flow_loss_det",
                    "qfx_grad_finalize_det", "qfx_fused_adamw_det"):
        getattr(L, fn_name).restype = C.c_int
    for i, (fn, msg) in enumerate(refusals):
        rc = fn()
        err = L.qfx_last_error().decode()
        assert rc == -1 and msg in err, (i, rc, err)


def test_emulated_entry_points_refuse_a_short_scratch(emu):
    with pytest.raises(AssertionError):
        emu.flow_loss_det(torch.zeros(1, 4, 64).bfloat16(), torch.zeros(1, 4, 64).bfloat16(), torch.zeros(1, 4, 64).bfloat16(), None,
                          1.0, torch.zeros(1), scratch=torch.zeros(295))
    with pytest.raises(AssertionError):
        emu.lora_wgrad_tc_det(torch.zeros(512, 256).bfloat16(), torch.zeros(512, 64).bfloat16(), [torch.zeros(256 * 16)], 16, 1, 16,
                              scratch=torch.zeros(256 * 16 * 2 - 1))


# ------------------------------------------------------------------------------------------------------------------ GPU
def _case(name):
    r = subprocess.run([sys.executable, CHECK, "--case", name], capture_output=True, text=True, timeout=1800,
                       env=dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8"))
    res = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
    assert r.returncode == 0 and res, (r.stdout + r.stderr)[-3000:]
    out = json.loads(res[-1][7:])
    print(name, out)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["attn_kernels", "reductions", "graph_and_recompute", "fp8_vs_bf16", "nf4_vs_bf16"])
def test_deterministic_kernels_and_exact_equalities(name):
    out = _case(name)
    assert not out.get("fail")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["r2r_qwen_ragged_b2", "r2r_qwen_edit_plus", "r2r_qwen_multires", "r2r_flux_yaml"])
def test_two_processes_give_the_same_digests(name):
    a, b = _case(name), _case(name)
    for k in ("loss_sha", "g32_sha", "lora_sha"):
        assert a[k] == b[k], (k, a, b)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["qwen_all_r4_b3", "qwen_all_r64", "qwen_subset_r16", "qwen_mod_embed_r4", "qwen_multires",
                                  "qwen_edit_plus_3img", "flux_all", "flux_yaml_targets", "flux_multires", "qwen_full_width_1blk",
                                  "flux_full_width_1p1"])
def test_lora_grads_keep_their_accuracy_under_the_flag(name):
    out = _case(f"lora_grad_{name}")
    assert not out["fail"] and out["det_attn_bwd_calls"] > 0
