"""The no-grad forward and the sampling loops at full depth against the block-streamed fp64 oracle, and validation between training
steps bit for bit (tools/infer_check.py).

CPU, with tests/emu_lib.py (and tests/det_ref.py) in place of the kernels at tiny depth and width:
  * every infer_check case runs end to end and passes (on the host the GraphCache runs eagerly; the workspace LRU still evicts);
  * the checks have teeth: a 1 % scale of one 128-row band of one sample's prediction is flagged, naming that sample and band, and
    nothing else is; a one-ulp change to one LoRA element of model B fails the validation check;
  * the no-grad forward reads no activation it did not write in the same call: with every activation buffer of every inference
    workspace filled with NaN before each call of a validation round, the round's latents do not change by one bit;
  * the dtype-generic oracle wrapper in fp64 on a monolithic tiny oracle equals the streamed one for a whole sampling loop.
GPU (`-m gpu`): every infer_check case at full depth, each in its own process."""
import copy
import json
import os
import subprocess
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, HERE)
CHECK = os.path.join(ROOT, "tools", "infer_check.py")

import infer_check as ic  # noqa: E402
import lora_grad_check as lg  # noqa: E402

F64 = torch.float64
CPU = torch.device("cpu")


@pytest.fixture()
def emu():
    import det_ref  # tests/emu_lib.py plus the deterministic entry points the validation case's training steps take
    from qflux_b200 import lib
    restore = det_ref.install(lib)
    yield lib
    restore()


QWEN_TINY = dict(layers=3, heads=2)
FLUX_TINY = dict(layers=2, single=2, heads=2)
# 8 x 12 patches: 192 image rows per sample, two 128-row bands, the first straddling the target / control boundary at row 96
TINY_ROUND = [((4, 6), 16, 8), ((6, 4), 12, 6), ((4, 4), 8, 16), ((2, 6), 10, 5)]
TINY = {
    "qwen_edit": dict(tiny=QWEN_TINY, cfg_update=dict(T=16, imgs=[(1, 4, 4)] * 2)),
    "qwen_edit_832x576": dict(tiny=QWEN_TINY, hw=(8, 12), T=16, T_neg=8),
    "flux_kontext_832x576": dict(tiny=FLUX_TINY, hw=(8, 12), T=16, T_neg=8),
    "qwen_plus": dict(tiny=QWEN_TINY, cfg_update=dict(T=16, imgs=[(1, 4, 4)] * 3)),
    "qwen_multires": dict(tiny=QWEN_TINY, cfg_update=dict(T=16)),
    "validation_qwen_edit": dict(tiny=QWEN_TINY, cfg_update=dict(T=16, imgs=[(1, 4, 4)] * 2), spec=TINY_ROUND),
    "validation_flux_kontext": dict(tiny=FLUX_TINY, cfg_update=dict(T=16, imgs=[(1, 4, 4)] * 2), spec=TINY_ROUND),
}


def _summary(res):
    return json.dumps(res, default=str)


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("name", list(ic.CASES))
def test_infer_check_wiring_on_cpu(emu, monkeypatch, name):
    import bench
    assert set(TINY) == set(ic.CASES)
    monkeypatch.setattr(bench, "MULTIRES_HW", [8, 4])  # the multi-resolution batch at tiny size: 128 and 32 image rows
    res = ic.CASES[name](dev=CPU, **TINY[name])
    print(name, _summary(res))
    assert not res["fail"], res["fail"]
    if name.startswith("validation"):
        assert res["round_shapes"] >= 8 and res["state_identical"]
        assert res["infer_workspaces_after_round"] == 3  # the LRU evicted: 8 shapes went through 3 workspaces
        assert res["round_repeat_identical"] and res["round_graphs_vs_eager_identical"] and res["round_finite"]
        return
    assert res["nograd_equals_grad_enabled"] and res["replay_equals_eager"]
    assert len(res["samples"]) == res["B"]
    if name.endswith("832x576"):
        assert [s["bands"] for s in res["samples"]] == [2, 2]
        assert len(res["sampler"]["samples"]) == 2
    if name == "qwen_multires":
        assert res["image_rows"] == [128, 32] and res["padded_rows_max_abs"] == 0.0


def test_one_band_scaled_by_one_percent_is_flagged(emu):
    """Band 1 of sample 1 holds control rows only, so the per-sample check over the target tokens is not touched by it."""
    res = ic.CASES["qwen_edit_832x576"](dev=CPU, corrupt=(1, 1, 1.01), sampling=False, **TINY["qwen_edit_832x576"])
    assert [f.split(":")[0] for f in res["fail"]] == ["sample 1 band 1"], res["fail"]
    assert res["samples"][1]["worst_band"]["band"] == 1


@pytest.mark.parametrize("name", ["validation_qwen_edit", "validation_flux_kontext"])
def test_one_ulp_in_one_lora_element_fails_validation(emu, name):
    res = ic.CASES[name](dev=CPU, nudge="transformer_blocks.0.attn.to_q.lora_B.default.weight", **TINY[name])
    assert res["fail"] and all(f.startswith("validation: training state after step 6 differs") for f in res["fail"]), res["fail"]
    assert not res["state_identical"]


@pytest.mark.parametrize("name", ["validation_qwen_edit", "validation_flux_kontext"])
def test_inference_reads_no_stale_activation(emu, name):
    """Round 2 runs with every activation buffer of every inference workspace NaN-filled before each forward: bit-identical latents."""
    res = ic.CASES[name](dev=CPU, poison=True, **TINY[name])
    assert not res["fail"], res["fail"]
    assert res["round_repeat_identical"] and res["round_finite"]


def test_poison_reaches_the_workspaces(emu):
    """The poisoning fills the activation buffers the forward reads and leaves the per-shape tables alone."""
    from qflux_b200 import sampler
    _, m = lg.qwen_pair(CPU, L=2, targets=lg.QWEN_ALL)
    names = ic._record_fixed_names(m)
    e = ic.sampler_batch("qwen", 1, (4, 4), 8, 8, m.J, steps=2)
    with torch.inference_mode():
        sampler.sample_qwen(m, e)
    assert names and len(m._infer_ws) == 1
    ws = next(iter(m._infer_ws.values()))
    ic._Poisoned(m, names).poison()
    assert bool(torch.isnan(ws["X"]).all()) and bool(torch.isnan(ws["dbl"][0]["qkv"]).all())
    assert all(bool(torch.isnan(t).all()) for t in ws["loraT"].values())
    assert torch.isfinite(ws["rope"]).all()


@pytest.mark.parametrize("family", ["qwen", "flux"])
def test_fp64_oracle_wrapper_streamed_equals_monolithic_sampling(family):
    """The dtype-generic wrapper in fp64: a whole true-CFG sampling loop on the monolithic tiny oracle and on the streamed oracle of the
    fused model holding the same weights gives the same latents."""
    from oracle import streamed
    from qflux_b200 import sampler
    if family == "qwen":
        orc, m = lg.qwen_pair(CPU, L=3, targets=lg.QWEN_ALL)
        e = ic.sampler_batch("qwen", 2, (4, 6), 12, 7, 128, steps=3)
        run = sampler.sample_qwen
    else:
        orc, m = lg.flux_pair(CPU, L=2, Ls=2, targets=lg.FLUX_ALL)
        e = ic.sampler_batch("flux", 2, (4, 6), 12, 7, 64, Pp=64, steps=3)
        run = sampler.sample_flux
    mono = ic.OracleModule(copy.deepcopy(orc).double(), F64, CPU)
    strm = ic.OracleModule(streamed.streamed_oracle(m, F64, CPU), F64, CPU)
    a, b = run(mono, e), run(strm, e)
    assert a.dtype == torch.bfloat16 and a.shape == (2, 24, 64)
    assert ic.same_bits(a, b)
    assert not ic.same_bits(a, e["latents"])


# ------------------------------------------------------------------------------------------------------------------ GPU
def _run_case(name):
    r = subprocess.run([sys.executable, CHECK, "--case", name], capture_output=True, text=True, timeout=1800, cwd=ROOT)
    res = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
    assert r.returncode == 0 and res, (r.stdout + r.stderr)[-3000:]
    out = json.loads(res[-1][7:])
    print(f"INFER_CHECK {name} " + json.dumps(out))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ic.CASES))
def test_full_depth_inference_on_gpu(name):
    out = _run_case(name)
    assert not out["fail"], out["fail"]
    if name.startswith("validation"):
        assert out["state_identical"] and out["train_graph_kept"] and out["round_repeat_identical"]
        assert out["round_graphs_vs_eager_identical"] and out["round_shapes"] >= 8
    else:
        assert out["graphs_captured"] == 1 and out["nograd_equals_grad_enabled"] and out["replay_equals_eager"]
