"""The joint attention backward keeps its bits (tools/attn_bwd_golden.py, tests/golden/attn_bwd_bits.json): SHA-256 of dK and dV
from qfx_attn_bwd, of dK, dV and dQ from qfx_attn_bwd_det, and of three deterministic FusedLoraAdamW steps, as recorded on one
device model.  On the CPU: the case list and the seeded inputs regenerate to what the JSON records.  On the GPU: every hash, on
the device model the goldens were recorded on (any other device skips: the step hashes depend on its SM count)."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import attn_bwd_golden as abg  # noqa: E402

with open(abg.GOLDEN) as _f:
    GOLD = json.load(_f)


def _on_golden_device():
    d = abg.device()
    if d != GOLD["device"]:
        pytest.skip(f"goldens were recorded on {GOLD['device']}, this device is {d}")


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_case_list_matches_golden():
    assert list(GOLD["cases"]) == [c[0] for c in abg.CASES]
    for name, B, H, S, split, txt, kv in abg.CASES:
        g = GOLD["cases"][name]
        assert (g["B"], g["H"], g["S"], g["split"], g["txt_len"], g["kv_len"]) == (B, H, S, split, txt, kv), name
    assert {n: (s["B"], s["txt_len"]) for n, s in GOLD["steps"].items()} == {n: (B, txt) for n, B, txt in abg.STEP_CASES}


@pytest.mark.parametrize("case", abg.CASES, ids=[c[0] for c in abg.CASES])
def test_seeded_inputs_match_golden(case):
    """the CPU-drawn inputs are reproducible (two draws agree) and are the ones the hashes were recorded from"""
    assert abg.inputs_sha(case) == abg.inputs_sha(case) == GOLD["cases"][case[0]]["inputs_sha"]


def test_cases_reach_the_mask_edges():
    """txt_len and kv_len at 63, 64, 65, 127, 128 and 129; S one below and above 128 boundaries; a fully masked key tile and a
    padding query tile"""
    edges = [63, 64, 65, 127, 128, 129]
    assert any(txt == edges for _, _, _, _, _, txt, _ in abg.CASES)
    assert any(kv == edges for *_, kv in abg.CASES)
    assert {383, 385, 639, 641} <= {S for _, _, _, S, *_ in abg.CASES}
    masked_tile = pad_tile = False
    for _, B, H, S, split, txt, kv in abg.CASES:
        for b in range(B):
            t = split if txt is None else txt[b]
            k = S if kv is None else kv[b]
            masked_tile |= any(k0 >= t and k0 + 128 <= split for k0 in range(0, S, 128))
            pad_tile |= (k + 63) // 64 < (S + 63) // 64
    assert masked_tile and pad_tile


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("case", abg.CASES, ids=[c[0] for c in abg.CASES])
def test_attention_backward_bits(case):
    _on_golden_device()
    got = abg.kernel_case(case)
    want = {k: v for k, v in GOLD["cases"][case[0]].items() if k.startswith(("atomic_", "det_"))}
    assert got == want


@pytest.mark.gpu
@pytest.mark.parametrize("name", [c[0] for c in abg.STEP_CASES])
def test_deterministic_step_bits(name):
    _on_golden_device()
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "attn_bwd_golden.py"), "--step", name], capture_output=True,
                       text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    want = {k: v for k, v in GOLD["steps"][name].items() if k.endswith("_sha")}
    assert got == want
