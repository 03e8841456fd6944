"""The joint attention forward / backward per row at the mask and tile edges the training step reaches (tools/attn_check.py: each
case against an fp64 reference scaled by bf16 SDPA, exact zeros where keys are masked, sentinels and tests/emu_lib.py), plus the
CPU-side checks that need no GPU: the fp64 reference agrees with the oracle's attention and with emu_lib under every mask
combination, and the C ABI refuses bad arguments before any CUDA call."""
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import attn_check as ac  # noqa: E402


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ac.CASES))
def test_attention_case(name):
    r = ac.CASES[name]()
    print(f"ATTN {name} " + json.dumps(r))
    assert not r["fail"], r["fail"]


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("masks", ["none", "txt", "kv", "both"])
def test_fp64_attention_reference_agrees_with_oracle_and_emulation(masks):
    """The reference the GPU cases trust, checked on CPU first, at split / kv_len on and next to the 64 / 128 tile edges: forward
    against the oracle's SDPA (an additive key mask, as the reference model builds it) and emu_lib, lse against logsumexp, the
    backward against fp64 autograd of the oracle's attention; emu_lib differs by bf16 rounding only, per row."""
    import torch
    import emu_lib as emu
    from oracle.mmdit_oracle import sdpa
    B, H, S, split = 4, 2, 257, 64
    Q, K, V, dO = (ac._mk(B, H, S, 128, seed=i, device="cpu") for i in range(4))
    kv = torch.tensor([65, 192, 193, 257], dtype=torch.int32) if masks in ("kv", "both") else None
    txt = torch.tensor([1, 63, 64, 0], dtype=torch.int32) if masks in ("txt", "both") else None
    mask = ac.key_mask(B, S, split, kv, txt)
    qv = torch.ones(B, S, dtype=torch.bool) if kv is None else torch.arange(S)[None] < kv[:, None]
    dO = dO * qv[:, None, :, None].to(dO.dtype)
    scale = 128 ** -0.5
    ref = ac.attn_ref(Q, K, V, mask, scale, dO)
    add = torch.zeros(B, 1, 1, S, dtype=torch.float64).masked_fill(~mask[:, None, None, :], float("-inf"))
    q, k, v = (t.double().transpose(1, 2).requires_grad_(True) for t in (Q, K, V))
    o = sdpa(q, k, v, add)  # [B, S, H, 128]
    assert torch.allclose(ref["O"], o.detach().transpose(1, 2), atol=1e-10)
    gq, gk, gv = torch.autograd.grad(o, (q, k, v), dO.double().transpose(1, 2))
    for name, g in (("dQ", gq), ("dK", gk), ("dV", gv)):
        assert torch.allclose(ref[name], g.transpose(1, 2), atol=1e-10), name
    s = (Q.double() @ K.double().transpose(-1, -2) * scale).masked_fill(~mask[:, None, None, :], float("-inf"))
    assert torch.allclose(ref["lse"], torch.logsumexp(s, -1) * ac.LOG2E, atol=1e-10)
    # masked keys get no gradient; dQ rows past kv_len none (their dO is zero)
    assert (ref["dK"][~mask[:, None, :].expand(B, H, S)] == 0).all() and (ref["dV"][~mask[:, None, :].expand(B, H, S)] == 0).all()
    assert (ref["dQ"][~qv[:, None, :].expand(B, H, S)] == 0).all()
    # emu_lib, row by row
    ot, oi, le = torch.empty(B * split, H * 128, dtype=torch.bfloat16), torch.empty(B * (S - split), H * 128, dtype=torch.bfloat16), torch.empty(B, H, S)
    emu.attn_fwd(Q, K, V, ot, oi, split, le, kv_len=kv, scale=scale, txt_len=txt)
    Oe = ac._o_headmajor(ot, oi, B, H, S, split)
    assert ac._rowerr(Oe, ref["O"]).max() < 1e-2
    assert (le.double() - ref["lse"]).abs().max() < 1e-4
    delta = (dO.float() * Oe.float()).sum(-1)
    dq, dk, dv = torch.zeros(B, H, S, 128), torch.empty(B, H, S, 128, dtype=torch.bfloat16), torch.empty(B, H, S, 128, dtype=torch.bfloat16)
    emu.attn_bwd(Q, K, V, dO, le, delta, dq, dk, dv, kv_len=kv, scale=scale, txt_len=txt, split=split)
    sel = qv[:, None, :].expand(B, H, S)
    assert ac._rowerr(dq, ref["dQ"], ref["dQ_mag"])[sel].max() < 2e-2
    assert ac._rowerr(dk, ref["dK"], ref["dK_mag"])[mask[:, None, :].expand(B, H, S)].max() < 2e-2
    assert ac._rowerr(dv, ref["dV"])[mask[:, None, :].expand(B, H, S)].max() < 2e-2
    # the eager scale the GPU cases use: bf16 SDPA with the same boolean mask
    eag = ac.attn_eager(Q, K, V, mask, scale, dO)
    assert ac._rowerr(eag["O"], ref["O"]).max() < 3e-2


def test_padding_tile_rows():
    """the forward's padding tiles: 128-row query tiles starting at or past both kv_len[b] and split"""
    import torch
    pad = ac.padding_tile_rows(3, 400, 129, torch.tensor([130, 256, 400]))
    assert pad[0].nonzero().flatten().tolist() == list(range(256, 400))
    assert pad[1].nonzero().flatten().tolist() == list(range(256, 400))
    assert not pad[2].any()
    assert not ac.padding_tile_rows(1, 400, 300, torch.tensor([140]))[0, :256].any()


def _err(lib):
    return lib._lib.qfx_last_error().decode()


def test_attention_refuses_bad_arguments_without_gpu():
    """The attention entry points check their row groups, strides, alignment and the text-mask split before any CUDA call: each
    refusal comes back with its message on a machine without a driver."""
    from qflux_b200 import lib
    P = 0x10000
    B, H, S, split = 2, 2, 300, 44
    D = H * 128

    def fwd(out0=P, ld0=D, rows0=split, out1=P, ld1=D, rows1=S - split, sp=split, txt=0):
        return lib._attn_fwd(P, P, P, out0, ld0, rows0, out1, ld1, rows1, sp, P, 0, txt, B, H, S, 0.088, None)

    def bwd(sp=split, txt=P, dQ=P, dK=P, dV=P):
        return lib._attn_bwd(P, P, P, P, P, P, dQ, dK, dV, 0, txt, sp, B, H, S, 0.088, None)

    refusals = [
        (lambda: fwd(rows0=split - 1), "row groups too short"), (lambda: fwd(rows1=S - split - 1), "row groups too short"),
        (lambda: fwd(sp=-1), "row groups too short"),
        (lambda: fwd(sp=0, rows1=S, txt=P), "txt_len needs 0 < split <= S"),
        (lambda: fwd(ld0=D + 4), "16-byte aligned"), (lambda: fwd(ld1=D + 2), "16-byte aligned"),
        (lambda: fwd(ld0=D - 128), "16-byte aligned"), (lambda: fwd(out1=P + 4), "16-byte aligned"),
        (lambda: fwd(out0=P + 8), "16-byte aligned"),
        (lambda: bwd(sp=0), "txt_len needs 0 < split <= S"), (lambda: bwd(sp=S + 1), "txt_len needs 0 < split <= S"),
        (lambda: bwd(dQ=P + 4), "dQ_accum must be 8-byte aligned"), (lambda: bwd(dK=P + 2), "dQ_accum must be 8-byte aligned"),
        (lambda: bwd(dV=P + 1), "dQ_accum must be 8-byte aligned"),
    ]
    for i, (fn, msg) in enumerate(refusals):
        rc = fn()
        assert rc != 0 and msg in _err(lib), (i, msg, _err(lib))
    import torch
    if not torch.cuda.is_available():  # valid calls get past every check and stop where the driver is needed
        for fn in (lambda: fwd(), lambda: fwd(sp=S, out1=0, rows0=S), lambda: bwd(), lambda: bwd(sp=0, txt=0)):
            rc = fn()
            assert rc != 0 and "cuTensorMapEncodeTiled" in _err(lib), _err(lib)
