"""4-bit NF4 base checkpoints (qflux_b200/nf4.py, DESIGN.md §3): the bitsandbytes state-dict form, NF4-resident block weights
dequantized block by block into the two-slot ring, and the refusals.

CPU (emulated kernels, tests/emu_lib.py + tests/nf4_ref.py): the loader against an independent restatement of bitsandbytes'
quantizer / `dequantize_4bit`, and bit-identical loss, prediction and LoRA gradients between an NF4 model and a bf16 model loaded
with the dequantized weights.  GPU (one subprocess per case, tools/nf4_check.py): the kernel bit for bit at full size, full-depth
Qwen-Image-Edit parity, CUDA-graph replay of the NF4 ring and the memory it frees."""
import importlib.util
import os
import subprocess
import sys

import pytest
import torch

import nf4_ref
import test_activation_recompute as tar

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
QWEN_TARGETS = ("to_q", "to_k", "to_v", "to_out.0", "add_q_proj", "img_mod.1", "txt_mod.1", "img_mlp.net.2", "txt_mlp.net.0.proj",
                "img_in", "txt_in")


@pytest.fixture()
def emu():
    from qflux_b200 import lib
    restore = nf4_ref.install(lib)
    yield lib
    restore()


def _in_blocks(mod):
    return mod.startswith(("transformer_blocks.", "single_transformer_blocks."))


def _every_linear(mod):
    return True


def _bf16_model(family, **kw):
    return tar._qwen(**kw) if family == "qwen" else tar._flux(**kw)


def _pair(family, nested=False, storage=torch.uint8, key=lambda k: k, select=_every_linear, **kw):
    """(NF4 model, bf16 model holding the dequantized weights, NF4 state dict) with identical adapters."""
    src = _bf16_model(family, **kw)
    base = {k: v for k, v in src.state_dict().items() if ".lora_" not in k}
    base = {k.replace(".base_layer.", "."): v for k, v in base.items()}
    qsd = nf4_ref.to_nf4_state_dict(base, select, nested=nested, storage=storage, key=key)
    deq = {}
    for k, v in base.items():
        kk = key(k)
        deq[k] = nf4_ref.dequantize_4bit(qsd, kk) if kk + ".quant_state.bitsandbytes__nf4" in qsd else v
    cls, cfg = type(src), src.config
    lora = {k: v for k, v in src.state_dict().items() if ".lora_" in k}
    models = []
    for fw, sd in (("nf4", qsd), ("bf16", deq)):
        m = cls(cfg, device="cpu", _host_only=True, frozen_weights=fw)
        targets = src.peft_config[src.adapter_name].target_modules
        m.add_adapter(src.lora_rank, src.lora_rank * src.lora_scaling, target_modules=targets)
        m.load_state_dict({**sd, **lora}, strict=True)
        models.append(m)
    return models[0], models[1], qsd


def _same_step(a, b):
    tar._same(a, b)


# ------------------------------------------------------------------------------------------------------------------ format
@pytest.mark.parametrize("nested", [False, True])
@pytest.mark.parametrize("storage", [torch.uint8, torch.bfloat16])
def test_loader_matches_the_restated_dequantization(nested, storage):
    from qflux_b200 import nf4
    g = torch.Generator().manual_seed(1)
    W = torch.randn(96, 320, generator=g) * 0.05
    W[3, :64] = 0  # an all-zero quantization block
    ent = {"blk.lin.weight" + s: t for s, t in nf4_ref.quantize_nf4(W, 64, nested, storage, nested_blocksize=32).items()}
    plain, quant = nf4.split_state_dict({**ent, "blk.lin.bias": torch.zeros(96)})
    assert list(plain) == ["blk.lin.bias"] and list(quant) == ["blk.lin.weight"]
    ours = nf4.dequantize(quant["blk.lin.weight"])
    assert torch.equal(ours, nf4_ref.dequantize_4bit(ent, "blk.lin.weight"))
    assert (ours.float() - W).abs().max() < 0.04  # a sanity bound on the restated quantizer, not part of the contract


@pytest.mark.skipif(importlib.util.find_spec("bitsandbytes") is None, reason="bitsandbytes is not installed")
@pytest.mark.parametrize("nested", [False, True])
def test_restatement_against_bitsandbytes(nested):
    """Pins the serialized layout and the dequantization rule wherever the package exists."""
    import bitsandbytes as bnb
    from qflux_b200 import nf4
    if not torch.cuda.is_available():
        pytest.skip("bitsandbytes quantizes on a CUDA device")
    lin = bnb.nn.Linear4bit(256, 128, compute_dtype=torch.bfloat16, compress_statistics=nested, quant_type="nf4")
    lin.load_state_dict({"weight": torch.randn(128, 256) * 0.05, "bias": torch.zeros(128)})
    lin = lin.cuda()
    sd = {"m." + k: v for k, v in lin.state_dict().items()}
    _, quant = nf4.split_state_dict(sd)
    ref = bnb.functional.dequantize_4bit(lin.weight.data, lin.weight.quant_state).to(torch.bfloat16).cpu()
    assert torch.equal(nf4.dequantize(quant["m.weight"]), ref)
    assert torch.equal(nf4_ref.dequantize_4bit({k: v.cpu() for k, v in sd.items()}, "m.weight"), ref)


@pytest.mark.parametrize("nested,storage,prefix", [(False, torch.uint8, ""), (True, torch.uint8, "base_layer"),
                                                   (True, torch.bfloat16, "transformer"), (False, torch.bfloat16, "both")])
def test_fused_model_holds_the_dequantized_weights(emu, nested, storage, prefix):
    def key(k):
        if prefix in ("base_layer", "both") and _in_blocks(k):
            k = k[: -len(".weight")] + ".base_layer.weight" if k.endswith(".weight") else k
        return ("transformer." + k) if prefix in ("transformer", "both") else k
    m, ref, qsd = _pair("qwen", nested, storage, key, L=2)
    assert m.frozen_weights == "nf4" and ref.frozen_weights == "bf16"
    # every block matrix, dequantized through the ring, equals the restated dequantize_4bit
    views = ref._weight_views()
    for blk in range(m.L):
        m._acquire(blk, -1)
        for k, v in m._weight_views(store=True).items():
            if k.startswith(f"transformer_blocks.{blk}.") and v.is_meta:
                kind = m._matrix_kind(k)
                got = m.w[kind][blk].reshape(-1)[v.storage_offset() - blk * m.w[kind].numel:][: v.numel()].view(v.shape)
                assert torch.equal(got, views[k]), k
        m._release(blk)
    # outside the blocks the model keeps bf16, dequantized at load
    for k, wk in (("img_in.weight", "img_in_w"), ("txt_in.weight", "txt_in_w"), ("proj_out.weight", "proj_out_w"),
                  ("norm_out.linear.weight", "norm_out_w"), ("time_text_embed.timestep_embedder.linear_1.weight", "t1_w")):
        assert torch.equal(m.w[wk], views[k]) and m.w[wk].dtype == torch.bfloat16, k


def test_frozen_weight_bytes_are_the_computed_bytes(emu):
    m, ref, _ = _pair("flux", nd=2, ns=3)
    D, L, Ls = m.D, m.L, m.Ls
    params = L * 2 * (6 + 3 + 1 + 4 + 4) * D * D + Ls * (3 + 3 + 4 + 5) * D * D
    stored = sum(c.numel() * c.element_size() + a.numel() * a.element_size() for c, a in m._nf4_store.values())
    assert stored == params // 2 + params // 64 * 4
    slots = sum(r.gbuf.numel() * 2 for r in m._nf4_rings)
    assert slots == 2 * 2 * (2 * 18 * D * D + 15 * D * D)
    assert not any(torch.is_tensor(m.w[k]) for k in m._nf4_store)  # the bf16 stacks were never allocated


# ------------------------------------------------------------------------------------------------------------------ parity
@pytest.mark.parametrize("kind", ["dense", "plus", "multi"])
def test_qwen_nf4_equals_bf16_with_dequantized_weights(emu, kind):
    m, ref, _ = _pair("qwen", nested=True, select=_in_blocks, targets=QWEN_TARGETS)
    batch = tar._qwen_batch(kind)
    _same_step(tar._fused(m, "qwen", batch), tar._fused(ref, "qwen", batch))


@pytest.mark.parametrize("kind", ["dense", "multi"])
def test_flux_nf4_equals_bf16_with_yaml_targets(emu, kind):
    m, ref, _ = _pair("flux")
    assert any(k.startswith("single_") for k in m.mod_sites.get("sgl", {}).get("names", [])) and any(s[0] == -1 for s in m.sites)
    batch = tar._flux_batch(kind)
    _same_step(tar._fused(m, "flux", batch), tar._fused(ref, "flux", batch))


@pytest.mark.parametrize("family", ["qwen", "flux"])
@pytest.mark.parametrize("mode", ["partial", "all"])
def test_nf4_with_forced_recompute(emu, monkeypatch, family, mode):
    from qflux_b200 import mmdit_base
    monkeypatch.setattr(mmdit_base, "plan_activation_memory", tar.force_plan(mode))
    m, ref, _ = _pair(family)
    batch = (tar._qwen_batch if family == "qwen" else tar._flux_batch)("dense")
    _same_step(tar._fused(m, family, batch), tar._fused(ref, family, batch))
    assert m.activation_plan.recompute


@pytest.mark.parametrize("family", ["qwen", "flux"])
def test_nf4_gradient_accumulation_and_autograd_bridges(emu, family):
    m, ref, _ = _pair(family)
    mk = tar._qwen_batch if family == "qwen" else tar._flux_batch
    res = []
    for model in (m, ref):
        step = tar._step(model, family, gradient_accumulation_steps=2, use_cuda_graph=False)
        for seed in (0, 1):
            emb, noise, u = mk("dense", seed)
            step.train_step(emb, None, noise, u)
        gacc = model.G32.clone()
        emb, noise, u = mk("dense", 2)
        model.zero_grad()
        loss = step.compute_loss(emb, noise, u)  # step bridge
        loss.backward()
        g1 = [p.grad.clone() for p in model.parameters()]
        model.zero_grad()
        pred = _model_bridge_pred(model, family, mk("dense", 3))
        pred.float().square().mean().backward()  # model bridge (ModelFn)
        g2 = [p.grad.clone() for p in model.parameters()]
        res.append((gacc, g1, g2, pred.detach()))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][3], res[1][3])
    for a, b in zip(res[0][1] + res[0][2], res[1][1] + res[1][2]):
        assert torch.equal(a, b)


def _model_bridge_pred(model, family, batch):
    emb, noise, u = batch
    B = emb["image_latents"].shape[0]
    x = torch.cat([emb["image_latents"], emb["control_latents"]], 1)
    if family == "qwen":
        return model(x, emb["prompt_embeds"], None, u.to(torch.bfloat16), emb["img_shapes"])[0]
    ids = torch.cat([emb["image_ids"], emb["control_ids"]], 0)
    return model(x, emb["prompt_embeds"], emb["pooled_prompt_embeds"], u.to(torch.bfloat16), ids, emb["text_ids"],
                 torch.ones(B))[0]


@pytest.mark.parametrize("family", ["qwen", "flux"])
def test_nf4_no_grad_forward_and_sampler(emu, family):
    m, ref, _ = _pair(family)
    mk = tar._qwen_batch if family == "qwen" else tar._flux_batch
    with torch.no_grad():
        a, b = _model_bridge_pred(m, family, mk("dense", 4)), _model_bridge_pred(ref, family, mk("dense", 4))
    assert torch.equal(a, b)
    if family == "qwen":
        from qflux_b200.sampler import sample_qwen
        emb, noise, _ = mk("dense", 5)
        emb = dict(emb, latents=noise, prompt_embeds_mask=torch.ones(emb["prompt_embeds"].shape[:2], dtype=torch.int64),
                   num_inference_steps=2)
        assert torch.equal(sample_qwen(m, emb), sample_qwen(ref, emb))


def _shim_reference(family, nf4_sd, cfg):
    """A reference-like transformer whose `state_dict()` is in the bitsandbytes NF4 form (what a trainer built from a 4-bit
    config holds), optionally with a PEFT adapter."""
    class Ref(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.config = cfg

        def state_dict(self, *a, **k):
            return dict(nf4_sd)
    return Ref()


@pytest.mark.parametrize("family", ["qwen", "flux"])
def test_from_reference_and_patch_trainer_on_an_nf4_reference(emu, family):
    from qflux_b200 import integration
    m, ref, qsd = _pair(family, nested=True, key=lambda k: k[: -len(".weight")] + ".base_layer.weight"
                        if _in_blocks(k) and k.endswith(".weight") else k)
    cfg = {k: getattr(m.config, k) for k in m.config.__dataclass_fields__}
    dit = integration.from_reference(_shim_reference(family, qsd, cfg), _host_only=True)
    assert dit.frozen_weights == "nf4" and dit.nf4_blocksize == 64
    trainer = type("T", (), {})()
    trainer.dit = _shim_reference(family, qsd, cfg)
    integration.patch_trainer(trainer, _host_only=True)
    assert trainer.dit.frozen_weights == "nf4"
    for model in (dit, ref):
        model._lora_params.clear()
    dit.add_adapter(4, 4, target_modules=("to_q", "to_v"), b_std=0.05)
    ref2 = type(ref)(ref.config, device="cpu", _host_only=True)
    ref2.load_state_dict({k: v for k, v in ref.state_dict().items() if ".lora_" not in k}, strict=False)
    ref2.add_adapter(4, 4, target_modules=("to_q", "to_v"), b_std=0.05)
    batch = (tar._qwen_batch if family == "qwen" else tar._flux_batch)("dense")
    _same_step(tar._fused(dit, family, batch), tar._fused(ref2, family, batch))


def test_save_and_load_lora_on_an_nf4_model(emu, tmp_path):
    m, ref, _ = _pair("qwen")
    sd = m.state_dict()
    assert not any(k.startswith("transformer_blocks.") and ".lora_" not in k for k in sd)
    assert "img_in.base_layer.weight" in sd or "img_in.weight" in sd
    lora = {"transformer." + k.replace(".default", ""): v for k, v in sd.items() if ".lora_" in k}
    m2, _, qsd = _pair("qwen")
    m2._lora_params.clear()
    fresh = type(m)(m.config, device="cpu", _host_only=True, frozen_weights="nf4")
    fresh.load_state_dict({k: v for k, v in qsd.items()}, strict=False)
    fresh.load_lora_adapter(lora)
    assert all(torch.equal(fresh._lora_params[k], p) for k, p in m._lora_params.items())


# ------------------------------------------------------------------------------------------------------------------ refusals
def _one(W=None, **kw):
    W = torch.randn(64, 128) * 0.05 if W is None else W
    return {"transformer_blocks.0.attn.to_q.weight" + s: t for s, t in nf4_ref.quantize_nf4(W, **kw).items()}


def _edit_meta(ent, **upd):
    import json
    k = next(k for k in ent if k.endswith("bitsandbytes__nf4"))
    meta = json.loads(bytes(ent[k].tolist()).decode())
    meta.update(upd)
    ent = dict(ent)
    ent[k] = torch.tensor(list(json.dumps(meta).encode()), dtype=torch.uint8)
    return ent


def test_refuses_fp4_and_int8_and_bad_blocksizes_and_foreign_code_books():
    from qflux_b200 import lib, nf4
    ent = _one()
    fp4 = {k.replace("__nf4", "__fp4"): v for k, v in _edit_meta(ent, quant_type="fp4").items()}
    with pytest.raises(lib.QfxError, match="fp4"):
        nf4.split_state_dict(fp4)
    with pytest.raises(lib.QfxError, match="int8"):
        nf4.split_state_dict({"transformer_blocks.0.attn.to_q.weight": torch.zeros(64, 128, dtype=torch.int8),
                              "transformer_blocks.0.attn.to_q.SCB": torch.ones(64)})
    with pytest.raises(lib.QfxError, match="does not divide in_features"):
        nf4.split_state_dict(_one(torch.randn(64, 96), blocksize=64))
    bad = dict(ent)
    bad["transformer_blocks.0.attn.to_q.weight.quant_map"] = torch.linspace(-1, 1, 16)
    with pytest.raises(lib.QfxError, match="code book"):
        nf4.split_state_dict(bad)


def test_refuses_format_and_constructor_mismatches(emu):
    from qflux_b200 import lib
    m, ref, qsd = _pair("qwen", L=2)
    bf = type(m)(m.config, device="cpu", _host_only=True)
    with pytest.raises(lib.QfxError, match="frozen_weights='nf4'"):
        bf.load_state_dict(qsd)
    with pytest.raises(lib.QfxError, match="frozen_weights='bf16'"):
        type(m)(m.config, device="cpu", _host_only=True, frozen_weights="nf4").load_state_dict(ref.state_dict(), strict=False)
    # a stacked kind whose layers arrive in mixed formats (block 0 NF4, block 1 bf16)
    base = {k: v for k, v in ref.state_dict().items() if ".lora_" not in k}
    mixed = nf4_ref.to_nf4_state_dict(base, lambda mod: mod.startswith("transformer_blocks.0."))
    with pytest.raises(lib.QfxError, match="one format"):
        type(m)(m.config, device="cpu", _host_only=True, frozen_weights="nf4").load_state_dict(mixed)
    with pytest.raises(lib.QfxError, match="frozen_weights"):
        type(m)(m.config, device="cpu", _host_only=True, frozen_weights="int4")


def test_refuses_sharding_and_merge_adapter(emu):
    from qflux_b200 import lib
    m, _, _ = _pair("qwen", L=2)
    with pytest.raises(lib.QfxError, match="sharded NF4"):
        m.shard_frozen_weights()
    with pytest.raises(lib.QfxError, match="NF4-resident"):
        m.merge_adapter()


# ------------------------------------------------------------------------------------------------------------------ GPU
def _gpu_case(name):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "nf4_check.py"), name], capture_output=True, text=True, cwd=ROOT)
    print(r.stdout[-4000:], r.stderr[-4000:])
    assert r.returncode == 0, name


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["kernel_qwen_double", "kernel_flux_single", "qwen_full_parity", "graph_replay", "infer_replay"])
def test_gpu(name):
    _gpu_case(name)
