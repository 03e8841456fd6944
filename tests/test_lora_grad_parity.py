"""Every LoRA gradient tensor of the fused step against an fp64 oracle (tools/lora_grad_check.py): per tensor, the fused error must
stay within 1.5x the bf16-eager oracle's own error + 2e-3 and under 3e-2, on the autograd path, the `train_step` fast path and the
module-forward bridge; tensors the oracle never reaches must get exactly zero.  Plus the tiling of the flat gradient buffer and
the zero padding of every LoRA site after an optimizer step.

CPU: the host wiring (flat-buffer offsets, fused q|k|v slots, modulation row indices, per-sample loops) with tests/emu_lib.py in
place of the kernels.  GPU: the same cases on the real kernels, and full-width blocks that reach the kernels' large-shape paths."""
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import lora_grad_check as lg  # noqa: E402


@pytest.fixture()
def emu():
    import emu_lib
    from qflux_b200 import lib
    restore = emu_lib.install(lib)
    yield lib
    restore()


def _report(name, res):
    for path, rep in res["paths"].items():
        print(lg.format_table(f"{name} [{path}]", rep))


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", list(lg.TINY))
def test_lora_grads_per_tensor_on_cpu(emu, name):
    import torch
    res = lg.TINY[name](dev=torch.device("cpu"))
    _report(name, res)
    assert not res["fail"], res["fail"]


def test_per_tensor_check_catches_what_the_pooled_norm_hides(emu):
    """Two wrong small tensors — block 1's txt_mod.1 lora_A 10 % too large and block 0's to_q lora_A missing — are flagged by name,
    and only those, while the pooled relative L2 over all LoRA tensors stays under the 2e-2 the CPU step tests allow."""
    import torch
    res = lg.TINY["qwen_mod_embed_r4"](dev=torch.device("cpu"), keep=True)
    got, g64, g16 = res["paths"]["autograd"]["grads"]
    assert not lg.per_tensor(got, g64, g16)["fail"]
    bad = {"transformer_blocks.1.txt_mod.1.lora_A.default.weight": lambda g: g * 1.1,
           "transformer_blocks.0.attn.to_q.lora_A.default.weight": lambda g: torch.zeros_like(g)}
    mutated = {n: (bad[n](g) if n in bad else g) for n, g in got.items()}
    rep = lg.per_tensor(mutated, g64, g16)
    print(lg.format_table("mutated", rep))
    assert sorted(f.split(":")[0] for f in rep["fail"]) == sorted(bad), rep["fail"]
    assert rep["pooled"] < 2e-2, rep["pooled"]
    # a gradient where the oracle has none must be exactly zero
    some = next(iter(g64))
    rep = lg.per_tensor(got, {**g64, some: None}, g16)
    assert [f.split(":")[0] for f in rep["fail"]] == [some]


def test_invariant_checks_catch_overlap_and_dirty_padding(emu):
    """The tiling check sees two parameters sharing gradient storage; the padding check sees a non-zero row past the rank."""
    import torch
    orc, m = lg.qwen_pair(torch.device("cpu"), targets=("to_q", "to_v", "img_mod.1"))
    assert not lg.tiling_fail(m) and not lg.padding_fail(m)
    members = m._extra_members
    full, pA, pB, ga, gb, d_in, d_out = members[0]
    members[0] = (full, pA, pB, ga + 1, gb, d_in, d_out)
    assert lg.tiling_fail(m)
    members[0] = (full, pA, pB, ga, gb, d_in, d_out)
    site = m.sites[(0, "qkv", 0)]
    site.A_pad[64 + m.lora_rank, 0] = 1.0         # slot 1 (to_k) has no adapter: its whole A block is padding
    assert any("slot 1" in f for f in lg.padding_fail(m))
    site.A_pad.zero_()
    site.B_pad[0, m.lora_rank] = 1.0
    assert any("B_pad" in f for f in lg.padding_fail(m))


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(lg.TINY) + list(lg.FULL_WIDTH))
def test_lora_grads_per_tensor_on_gpu(name):
    fn = lg.TINY.get(name) or lg.FULL_WIDTH[name]
    res = fn()
    _report(name, res)
    print(f"{name}: worst ratio {res['worst_ratio']:.2f}")
    assert not res["fail"], res["fail"]
