"""The benchmarked training steps at full depth against a block-streamed fp64 oracle (tools/depth_check.py, oracle/streamed.py).

CPU:
  * the streamed oracle, run one sample at a time the way depth_check runs it, equals the monolithic `QwenImageOracle` / `FluxOracle`
    in fp64 (prediction, loss, every LoRA gradient) with LoRA on the block Linears, the modulation / AdaLN linears and the embedders:
    Qwen with 3 blocks, FLUX with 2 + 2 blocks, and one Qwen multi-resolution batch;
  * building the blocks consumes every key of the fused model's `state_dict()` exactly once, and each built block holds exactly the
    fused model's weights;
  * the oracle reads the fused model's weights when it runs: one changed element of the last block changes its output;
  * depth_check's case code runs end to end at tiny depth and width with tests/emu_lib.py in place of the kernels, and a 10 % error in
    one gradient tensor of the last block is flagged by name, and nothing else is.
GPU (`-m gpu`): every depth_check case at full depth, each in its own process (every case starts on an empty device)."""
import copy
import json
import os
import subprocess
import sys
from collections import Counter

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, HERE)
CHECK = os.path.join(ROOT, "tools", "depth_check.py")

import depth_check as dc  # noqa: E402
import lora_grad_check as lg  # noqa: E402

F64 = torch.float64
CPU = torch.device("cpu")


@pytest.fixture()
def emu():
    import emu_lib
    from qflux_b200 import lib
    restore = emu_lib.install(lib)
    yield lib
    restore()


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300))


def _assert_equal_runs(streamed, mono_loss, mono_preds, mono_grads, loss_tol=1e-12):
    """streamed = oracle_run's (loss, preds, grads); the monolithic run's loss, per-sample predictions and `.grad`s."""
    loss, preds, grads = streamed
    mono_loss = float(mono_loss.detach() if torch.is_tensor(mono_loss) else mono_loss)
    assert abs(loss - mono_loss) <= loss_tol * abs(mono_loss), (loss, mono_loss)
    assert len(preds) == len(mono_preds)
    for p, q in zip(preds, mono_preds):
        assert _rel(p, q) <= 1e-12
    assert set(grads) == set(mono_grads)
    for n, g in grads.items():
        ref = mono_grads[n]
        if ref is None:
            assert g is None or not bool(g.any()), n
            continue
        assert g is not None and _rel(g, ref) <= 1e-12, (n, None if g is None else _rel(g, ref))


def _mono_run(mono, B, sample_loss):
    """The monolithic oracle through the same per-sample losses, one backward over their sum."""
    losses, preds = zip(*(sample_loss(mono, F64, b) for b in range(B)))
    sum(losses).backward()
    return sum(float(l.detach().double()) for l in losses), [p.detach() for p in preds], {n: (None if p.grad is None else p.grad.detach())
                                                for n, p in mono.named_parameters() if p.requires_grad}


def _qwen_inputs(B, L, T, J, seed=0):
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, dtype=F64)
    return dict(image_latents=rn(B, L, 64), control_latents=rn(B, L, 64), prompt_embeds=rn(B, T, J) * 3,
                prompt_embeds_mask=torch.ones(B, T, dtype=torch.int64), noise=rn(B, L, 64), u=torch.tensor([0.5, 0.25, 0.125][:B]))


# ------------------------------------------------------------------------------------------------------------------ CPU
def test_streamed_qwen_equals_monolithic():
    from oracle import mmdit_oracle as mo
    orc, m = lg.qwen_pair(CPU, L=3, targets=lg.QWEN_ALL)
    B, hw = 2, 4
    x = _qwen_inputs(B, hw * hw, 24, 128)
    shapes = [[(1, hw, hw), (1, hw, hw)]] * B

    def sample_loss(o, dt, b):
        sl = slice(b, b + 1)
        loss, p = mo.qwen_compute_loss(o, x["image_latents"][sl], x["control_latents"][sl], x["prompt_embeds"][sl],
                                       x["prompt_embeds_mask"][sl], shapes[sl], noise=x["noise"][sl], u=x["u"][sl])
        return loss / B, p[0]

    got = dc.oracle_run(m, F64, CPU, B, sample_loss)
    _assert_equal_runs(got, *_mono_run(copy.deepcopy(orc).double(), B, sample_loss))
    # the batched recipe: the sum of the per-sample losses differs from its batch mean only by the recipe's own fp32 loss arithmetic
    # (qwen_compute_loss takes the mean of pred.float()); predictions and gradients agree to fp64 rounding
    mono = copy.deepcopy(orc).double()
    loss, pred = mo.qwen_compute_loss(mono, **x, img_shapes=shapes)
    loss.backward()
    grads = {n: p.grad for n, p in mono.named_parameters() if p.requires_grad}
    _assert_equal_runs(got, loss, list(pred.detach()), grads, loss_tol=2.0 ** -23)
    assert any(".img_mod.1.lora_" in n for n in grads) and any(n.startswith("txt_in.lora_") for n in grads)


def test_streamed_flux_equals_monolithic():
    from oracle import mmdit_oracle as mo
    from qflux_b200.train_step import FluxKontextStep
    orc, m = lg.flux_pair(CPU, L=2, Ls=2, targets=lg.FLUX_ALL)
    B, hw, T = 2, 4, 8
    g = torch.Generator().manual_seed(3)
    rn = lambda *s: torch.randn(*s, generator=g, dtype=F64)
    x0, ctrl, pooled, pe, noise = rn(B, hw * hw, 64), rn(B, hw * hw, 64), rn(B, 64), rn(B, T, 64), rn(B, hw * hw, 64)
    ids = (torch.zeros(T, 3), FluxKontextStep.latent_image_ids(hw, hw, "cpu", 0.0), FluxKontextStep.latent_image_ids(hw, hw, "cpu", 1.0))
    t = torch.tensor([0.5, 0.25], dtype=F64)

    def sample_loss(o, dt, b):
        sl = slice(b, b + 1)
        loss, p = mo.flux_compute_loss_shared(o, x0[sl], ctrl[sl], pooled[sl], pe[sl], *ids, noise=noise[sl], t=t[sl])
        return loss / B, p[0]

    got = dc.oracle_run(m, F64, CPU, B, sample_loss)
    mono = copy.deepcopy(orc).double()
    loss, pred = mo.flux_compute_loss_shared(mono, x0, ctrl, pooled, pe, *ids, noise=noise, t=t)
    loss.backward()
    grads = {n: p.grad for n, p in mono.named_parameters() if p.requires_grad}
    _assert_equal_runs(got, loss, list(pred.detach()), grads)
    for part in ("x_embedder.lora_", "context_embedder.lora_", "transformer_blocks.1.norm1.linear.lora_",
                 "single_transformer_blocks.1.norm.linear.lora_", "single_transformer_blocks.1.proj_out.lora_"):
        assert any(n.startswith(part) for n in grads), part


def test_streamed_qwen_multires_equals_monolithic():
    """A pad-to-max multi-resolution batch's per-sample recipe (un-padded runs, AttentionMaskMseLoss normalisation)."""
    orc, m = lg.qwen_pair(CPU, L=3, targets=lg.QWEN_ALL)
    shapes = [[(1, 4, 4), (1, 4, 4)], [(1, 2, 4), (1, 2, 4)]]
    lt, txt = [16, 8], [8, 5]
    x = _qwen_inputs(2, 16, 8, 128, seed=11)
    sig = torch.tensor([0.5, 0.75])

    def sample_loss(o, dt, b):
        n = lt[b]
        noisy = (1 - sig[b]) * x["image_latents"][b, :n] + sig[b] * x["noise"][b, :n]
        p = o(hidden_states=torch.cat([noisy, x["control_latents"][b, :n]], 0)[None], timestep=sig[b:b + 1],
              encoder_hidden_states=x["prompt_embeds"][b:b + 1, :txt[b]], encoder_hidden_states_mask=x["prompt_embeds_mask"][b:b + 1, :txt[b]],
              img_shapes=[shapes[b]], txt_seq_lens=[txt[b]])[0][0, :n]
        return ((p - (x["noise"][b, :n] - x["image_latents"][b, :n])) ** 2).mean(-1).sum() / (sum(lt) + 1e-12), p

    got = dc.oracle_run(m, F64, CPU, 2, sample_loss)
    _assert_equal_runs(got, *_mono_run(copy.deepcopy(orc).double(), 2, sample_loss))


@pytest.mark.parametrize("family", ["qwen", "flux"])
def test_every_state_dict_key_is_used_once(family):
    """The top level and the blocks together are built from every key of the fused state dict exactly once, and every block built
    holds the fused model's weights (cast to fp64) and the oracle's LoRA leaves, nothing else."""
    from oracle import streamed
    orc, m = (lg.qwen_pair(CPU, L=3, targets=lg.QWEN_ALL) if family == "qwen" else lg.flux_pair(CPU, L=2, Ls=2, targets=lg.FLUX_ALL))
    sd = m.state_dict()
    o = streamed.streamed_oracle(m, F64, CPU)
    assert Counter(streamed.source_keys(o)) == Counter(list(sd))
    top = o.state_dict()
    blocks = [b for lst in ("transformer_blocks", "single_transformer_blocks") for b in getattr(o, lst, ())]
    assert len(blocks) == (3 if family == "qwen" else 4)
    for k in o.stream_top_keys:
        assert torch.equal(top[k], sd[k].double()), k
    for blk in blocks:
        built = blk.build().state_dict()
        assert sorted(blk.prefix + k for k in built) == sorted(blk.source_keys())
        leaves = dict(blk.named_parameters())
        for k, v in built.items():
            assert v.dtype == F64 and torch.equal(v, sd[blk.prefix + k].double()), blk.prefix + k
            if ".lora_" in k:
                assert v.data_ptr() == leaves[k].data_ptr(), f"{blk.prefix + k} is not the persistent leaf"


@pytest.mark.parametrize("family", ["qwen", "flux"])
def test_oracle_reads_the_fused_weights_when_it_runs(family):
    """One element of the last block's frozen weight, changed in the fused model after the oracle was made, changes its output."""
    from oracle import mmdit_oracle as mo, streamed
    from qflux_b200.train_step import FluxKontextStep
    if family == "qwen":
        orc, m = lg.qwen_pair(CPU, L=3, targets=lg.QWEN_ALL)
        key = "transformer_blocks.2.img_mlp.net.2.base_layer.weight"
        x = _qwen_inputs(1, 16, 8, 128)
        run = lambda o: o(hidden_states=torch.cat([x["image_latents"], x["control_latents"]], 1), timestep=torch.tensor([0.5]),
                          encoder_hidden_states=x["prompt_embeds"], img_shapes=[[(1, 4, 4), (1, 4, 4)]], txt_seq_lens=[8])[0]
    else:
        orc, m = lg.flux_pair(CPU, L=2, Ls=2, targets=lg.FLUX_ALL)
        key = "single_transformer_blocks.1.proj_out.base_layer.weight"
        g = torch.Generator().manual_seed(5)
        rn = lambda *s: torch.randn(*s, generator=g, dtype=F64)
        ids = torch.cat([FluxKontextStep.latent_image_ids(4, 4, "cpu", 0.0), FluxKontextStep.latent_image_ids(4, 4, "cpu", 1.0)])
        inp = dict(hidden_states=rn(1, 32, 64), encoder_hidden_states=rn(1, 8, 64), pooled_projections=rn(1, 64),
                   timestep=torch.tensor([0.5]), img_ids=ids, txt_ids=torch.zeros(8, 3), guidance=torch.ones(1))
        run = lambda o: o(**inp)[0]
    o = streamed.streamed_oracle(m, F64, CPU)
    with torch.no_grad():
        before = run(o)
        assert torch.equal(before, run(o))
        w = m.state_dict()[key]
        old = w[0, 0].clone()
        w[0, 0] += 0.5
        after = run(o)
        w[0, 0] = old
        assert not torch.equal(before, after)
        assert torch.equal(before, run(o))
    assert isinstance(o, mo.QwenImageOracle if family == "qwen" else mo.FluxOracle)


TINY = {
    "qwen_edit": dict(tiny=dict(layers=3, heads=2), cfg_update=dict(T=16, imgs=[(1, 4, 4)] * 2)),
    "qwen_edit_b4_recompute": dict(tiny=dict(layers=3, heads=2), cfg_update=dict(T=16, imgs=[(1, 4, 4)] * 2)),
    "flux_kontext": dict(tiny=dict(layers=2, single=2, heads=2), cfg_update=dict(T=16, imgs=[(1, 4, 4)] * 2)),
    "qwen_plus": dict(tiny=dict(layers=3, heads=2), cfg_update=dict(T=16, imgs=[(1, 4, 4)] * 3)),
    "qwen_multires": dict(tiny=dict(layers=3, heads=2), cfg_update=dict(T=16)),
}
LAST_BLOCK_TENSOR = {"qwen": "transformer_blocks.2.attn.to_v.lora_B.default.weight",
                     "flux": "single_transformer_blocks.1.attn.to_v.lora_B.default.weight"}


@pytest.mark.parametrize("name", list(dc.CASES))
def test_depth_check_wiring_on_cpu(emu, monkeypatch, name):
    """depth_check's case end to end at tiny depth and width on emulated kernels: everything passes except one last-block gradient
    tensor made 10 % too large, which is flagged by name."""
    import bench
    assert set(TINY) == set(dc.CASES)
    monkeypatch.setattr(bench, "MULTIRES_HW", [4, 2])  # the multi-resolution batch at tiny size: 64 and 32 px
    bad = LAST_BLOCK_TENSOR["flux" if name.startswith("flux") else "qwen"]
    res = dc.CASES[name](dev=CPU, corrupt={bad: 1.1}, **TINY[name])
    print(name, json.dumps({k: v for k, v in res.items() if k != "adamw"}))
    assert [f.split(":")[0] for f in res["fail"]] == [bad], res["fail"]
    assert res["adamw"]["adamw"]["elements"] == res["lora_elements"]
    if name == "qwen_edit_b4_recompute":
        assert 0 < res["recomputed_blocks"] < res["blocks"]
    assert len(res["worst_ratio_per_block"]) == res["blocks"]


# ------------------------------------------------------------------------------------------------------------------ GPU
def _run_case(name):
    r = subprocess.run([sys.executable, CHECK, "--case", name], capture_output=True, text=True, timeout=1800, cwd=ROOT)
    res = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
    assert r.returncode == 0 and res, (r.stdout + r.stderr)[-3000:]
    out = json.loads(res[-1][7:])
    print(f"DEPTH_CHECK {name} " + json.dumps(out))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(dc.CASES))
def test_full_depth_on_gpu(name):
    out = _run_case(name)
    assert out["graphs_captured"] == 1
    assert not out["fail"], out["fail"]
