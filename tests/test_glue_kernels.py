"""The glue kernels of the training step through their stream-pair entry points (tools/glue_check.py: each case against an fp64
reference, bf16 eager and tests/emu_lib.py, per row group and per row), plus the CPU-side checks that need no GPU: the fp64
reference helpers agree with the oracle and with emu_lib, and the C ABI refuses bad arguments before any CUDA call."""
import json
import math
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import glue_check as gc  # noqa: E402


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(gc.CASES))
def test_glue_case(name):
    r = gc.CASES[name]()
    print(f"GLUE {name} " + json.dumps(r))
    assert not r["fail"], r["fail"]


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_fp64_references_agree_with_oracle_and_emulation():
    """The references the GPU cases trust, checked on CPU first: RoPE against the oracle's complex and real forms, the
    LayerNorm-modulate / q-k norm / timestep / flow references against emu_lib (which rounds like the kernels, so the two may
    differ by bf16 rounding only, per row)."""
    import torch
    import emu_lib as emu
    from oracle.mmdit_oracle import apply_rotary_emb_qwen, apply_rotary_emb_real, diffusers_rms_norm, timestep_sinusoid
    BF = torch.bfloat16
    # RoPE: pairs (2i, 2i+1) rotated like apply_rotary_emb_qwen (complex) and apply_rotary_emb_real (cos/sin interleaved)
    x = gc._mk(2, 9, 3, 128, device="cpu", dtype=torch.float32)
    ang = torch.rand(9, 64, generator=torch.Generator().manual_seed(0)) * 6.28
    cs = torch.stack([ang.cos(), ang.sin()], -1)
    mine = gc.rope_ref(x, cs[None, :, None])
    assert torch.allclose(mine, apply_rotary_emb_qwen(x, torch.polar(torch.ones_like(ang), ang)), atol=1e-6)
    cos, sin = ang.cos().repeat_interleave(2, -1), ang.sin().repeat_interleave(2, -1)
    assert torch.allclose(mine, apply_rotary_emb_real(x, cos, sin), atol=1e-6)
    assert torch.allclose(gc.rms_ref(x, x[0, 0, 0]), diffusers_rms_norm(x, x[0, 0, 0], gc.EPS), atol=1e-6)
    # LayerNorm + modulate, both row groups (second group far from the first)
    D, T, L, B = 256, 7, 34, 3
    xx, sh, sc, gt, rows, M, split = gc._ln_operands(D, T, L, B, "cpu")
    y = torch.empty_like(xx)
    emu.ln_modulate_fwd_pair(xx, y, (sh[0], sc[0], T), (sh[1], sc[1], L), split)
    y64 = gc.ln_mod_ref(xx.double(), rows(sh).double(), rows(sc).double())
    assert gc.row_rel(y, y64).max() < 1e-2 and gc.rel(y[split:], y64[split:]) < 5e-3 and gc.rel(y[:split], y64[:split]) < 5e-3
    # q/k norm + RoPE, per-sample table, both conventions
    for rm in (False, True):
        H = 2
        qkv, w, rope, S, tokens, split = gc._qk_operands(H, T, L, B, True, "cpu")
        Q, K, V = (torch.zeros(B, H, S, 128, dtype=BF) for _ in range(3))
        emu.qk_norm_rope_fwd_pair(qkv, (w["q0"], w["k0"], T, 0), (w["q1"], w["k1"], L, T), split, rope, Q, K, V, round_mid=rm)
        for q64, k64, v, n, off in gc._qk_fwd_ref(qkv.double(), {k: v.double() for k, v in w.items()}, rope.double(), T, L, B, H,
                                                  gc.rms_ref):
            for got, ref in ((Q, q64), (K, k64)):
                g2 = gc._token_major(got, B, n, off)
                assert gc.row_rel(g2, ref.reshape(B * n, -1)).max() < 1e-2
            assert torch.equal(gc._token_major(V, B, n, off), v.reshape(B * n, -1).to(BF))
    # timestep embedding: the fp64 restatement vs the oracle's fp32 one
    t = torch.tensor([0.0, 0.25, 1.0]).to(BF).float()
    ref, arg = gc.timestep_ref(t, 256, 1000.0)
    assert (ref - timestep_sinusoid(t, 256, 1000.0).double()).abs().max() < 1e-3
    out = torch.empty(3, 256, dtype=BF)
    emu.timestep_sinusoid(t, 1000.0, out)
    assert ((out.double() - ref).abs() <= gc.ulp_bf16(ref) + 2.0 ** -20 * arg.abs() + 2.0 ** -20).all()
    # the flow-matching rule: emu_lib's bf16 tensor arithmetic is the stated rounding rule, bit for bit
    x0, nz = gc._mk(3, 11, 64, seed=1, device="cpu"), gc._mk(3, 11, 64, seed=2, device="cpu")
    ctrl = gc._mk(3, 5, 64, seed=3, device="cpu")
    sigma = torch.tensor([0.999, 0.123, 0.0371])
    packed = torch.empty(3, 16, 64, dtype=BF)
    emu.flow_noisy_input(x0, nz, ctrl, sigma, packed)
    assert torch.equal(packed[:, :11], gc.flow_rule(x0, nz, sigma)) and torch.equal(packed[:, 11:], ctrl)
    assert not torch.equal(gc.flow_rule(x0, nz, sigma), gc.flow_rule(x0, nz, sigma.to(BF).float() + 1e-3))


def test_emulated_clear_dq_zeroes_only_what_it_reads():
    """qfx.h: with clear_dq the kernel zeroes the dQ positions it reads, so the accumulator is clean only when the two row groups
    cover every joint position.  The emulation follows the same rule (a gap keeps its values), so a caller that breaks the
    contract fails the same way under both."""
    import torch
    import emu_lib as emu
    B, H, T, L, gap = 2, 2, 3, 5, 2
    S = T + gap + L
    qkv = gc._mk(B * (T + L), 3 * H * 128, device="cpu")
    w = gc._mk(128, device="cpu", shift=1.0)
    rope = torch.stack([torch.ones(S, 64), torch.zeros(S, 64)], -1)
    dQ = torch.randn(B, H, S, 128)
    keep = dQ.clone()
    dK, dV = torch.zeros(B, H, S, 128, dtype=torch.bfloat16), torch.zeros(B, H, S, 128, dtype=torch.bfloat16)
    dqkv = torch.empty_like(qkv)
    emu.qk_norm_rope_bwd_pair(dQ, dK, dV, qkv, (w, w, T, 0), (w, w, L, T + gap), B * T, rope, dqkv, clear_dq=True)
    assert (dQ[:, :, :T] == 0).all() and (dQ[:, :, T + gap:] == 0).all()
    assert torch.equal(dQ[:, :, T:T + gap], keep[:, :, T:T + gap])


def _err(lib):
    return lib._lib.qfx_last_error().decode()


def test_pair_entry_points_refuse_bad_arguments_without_gpu():
    """Argument validation happens before any CUDA call: a missing second-group operand, an unsupported hidden size and
    misaligned leading dimensions / bases are refused with a message, never launched (a misaligned vector access would fault)."""
    from qflux_b200 import lib
    P = 0x10000  # a 16-byte aligned stand-in address: nothing is dereferenced before the checks
    D, M, split = 512, 64, 16
    ok_bwd = dict(dy=P, lddy=D, x=P, ldx=D, mean=P, rstd=P, scale=P, ldmod=6 * D, rpb=8, dres=P, lddres=D, dx=P, lddx=D, gate=P,
                  ldgate=6 * D, dxg=P, lddxg=D, M=M, D=D, split=split, scale1=P, gate1=P, rpb1=16)

    def ln_fwd(D=D, ldx=D, shift1=P, scale1=P, rpb1=16):
        return lib._ln_fwd2(P, ldx, P, D, P, P, 6 * D, 8, P, P, M, D, 1e-6, split, shift1, scale1, rpb1, None)

    def ln_bwd(**kw):
        a = dict(ok_bwd, **kw)
        return lib._ln_bwd2(a["dy"], a["lddy"], a["x"], a["ldx"], a["mean"], a["rstd"], a["scale"], a["ldmod"], a["rpb"], a["dres"],
                            a["lddres"], a["dx"], a["lddx"], a["gate"], a["ldgate"], a["dxg"], a["lddxg"], a["M"], a["D"], a["split"],
                            a["scale1"], a["gate1"], a["rpb1"], None)
    H = 2
    ld3 = 3 * H * 128

    def qk_fwd(ldqkv=ld3, qkv=P, wq1=P, tps1=16):
        return lib._qknr_fwd2(qkv, ldqkv, P, P, P, 0, P, P, P, M, 8, 0, 24, H, 1e-6, 1, split, wq1, P, tps1, 8, None)

    def qk_bwd(ldqkv=ld3, lddqkv=ld3, dqkv=P, dQ=P, wk1=P):
        return lib._qknr_bwd2(dQ, P, P, P, ldqkv, P, P, P, 0, dqkv, lddqkv, M, 8, 0, 24, H, 1e-6, 1, split, P, wk1, 16, 8, 0, None)

    def delta(ldo=H * 128, lddo=H * 128, O=P, tps1=16):
        return lib._delta2(O, ldo, P, lddo, P, P, M, 8, 0, 24, H, split, tps1, 8, None)

    refusals = [
        (lambda: ln_fwd(shift1=None), "second group"), (lambda: ln_fwd(rpb1=0), "second group"),
        (lambda: ln_fwd(D=768, ldx=768), "hidden size 768 unsupported"), (lambda: ln_fwd(D=300, ldx=304), "bad dims"),
        (lambda: ln_bwd(scale1=None), "second group"), (lambda: ln_bwd(gate1=None), "second group"),
        (lambda: ln_bwd(D=768, lddy=768, ldx=768, lddres=768, lddx=768, lddxg=768, ldmod=6 * 768, ldgate=6 * 768), "hidden size 768 unsupported"),
        (lambda: qk_fwd(wq1=None), "second group incomplete"), (lambda: qk_fwd(tps1=0), "second group incomplete"),
        (lambda: qk_bwd(wk1=None), "second group incomplete"),
        (lambda: delta(tps1=0), "second group incomplete"),
    ]
    for name in ("lddy", "ldx", "ldmod", "lddres", "lddx", "ldgate", "lddxg"):
        refusals.append((lambda name=name: ln_bwd(**{name: ok_bwd[name] + 4}), "leading dimensions must be multiples of 8"))
    for name in ("dy", "x", "scale", "scale1", "dres", "dx", "gate", "gate1", "dxg"):
        refusals.append((lambda name=name: ln_bwd(**{name: P + 8}), "16-byte aligned"))
    refusals += [(lambda: qk_fwd(ldqkv=ld3 + 2), "ldqkv"), (lambda: qk_fwd(qkv=P + 4), "8-byte aligned"),
                 (lambda: qk_bwd(ldqkv=ld3 + 2), "leading dimensions"), (lambda: qk_bwd(lddqkv=ld3 + 1), "leading dimensions"),
                 (lambda: qk_bwd(dqkv=P + 2), "8-byte aligned"), (lambda: qk_bwd(dQ=P + 8), "8-byte aligned"),
                 (lambda: delta(ldo=H * 128 + 2), "leading dimensions"), (lambda: delta(lddo=H * 128 + 1), "leading dimensions"),
                 (lambda: delta(O=P + 4), "8-byte aligned")]
    # each call must stop at a check (a missing one would launch on stand-in addresses); the message says which check
    for i, (call, msg) in enumerate(refusals):
        rc = call()
        assert rc != 0 and msg in _err(lib), (i, msg, _err(lib))


def test_rounding_flip_bound_helpers():
    import torch
    v = torch.tensor([1.0, 1.5, 0.75, -3.0, 1e-3], dtype=torch.float64)
    assert torch.equal(gc.ulp_bf16(v), torch.tensor([2.0 ** -7, 2.0 ** -7, 2.0 ** -8, 2.0 ** -6, 2.0 ** -17], dtype=torch.float64))
    nxt = (v.to(torch.bfloat16).view(torch.int16) + 1).view(torch.bfloat16).double()
    assert torch.equal((nxt - v.to(torch.bfloat16).double()).abs(), gc.ulp_bf16(v))
    assert math.isclose(gc.rel(torch.ones(4), torch.ones(4)), 0.0)
