"""float8-e4m3fn base checkpoints (qflux_b200/fp8.py, DESIGN.md §3): FP8-resident block weights expanded block by block into the
two-slot ring, the two forms block matrices arrive in, and the refusals.

CPU (emulated kernels, tests/emu_lib.py + tests/fp8_ref.py): the round-trip check, and bit-identical loss, prediction and LoRA gradients between an
FP8 model and a bf16 model loaded with the expanded weights.  GPU (one subprocess per case, tools/fp8_check.py): the kernel against
torch's conversion on every code and at full size, multi-block training-step parity, CUDA-graph replay of the FP8 ring."""
import os
import subprocess
import sys

import pytest
import torch

import fp8_ref
import test_activation_recompute as tar

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E4M3 = torch.float8_e4m3fn
QWEN_TARGETS = ("to_q", "to_k", "to_v", "to_out.0", "add_q_proj", "img_mod.1", "txt_mod.1", "img_mlp.net.2", "txt_mlp.net.0.proj",
                "img_in", "txt_in")


@pytest.fixture()
def emu():
    from qflux_b200 import lib
    restore = fp8_ref.install(lib)
    yield lib
    restore()


def _in_blocks(k):
    return k.startswith(("transformer_blocks.", "single_transformer_blocks."))


def _base_layer(k):
    return k[: -len(".weight")] + ".base_layer.weight" if _in_blocks(k) and k.endswith(".weight") else k


def _fp8_checkpoint(base, form="float8", key=lambda k: k):
    """(checkpoint, expanded): every 2-D weight of `base` stored as e4m3fn (form "float8") or as its bf16 upcast (form "bf16", what
    diffusers' from_pretrained(torch_dtype=bf16) holds), and the bf16 weights both stand for."""
    ckpt, expanded = {}, {}
    for k, v in base.items():
        if k.endswith(".weight") and v.ndim == 2:
            c = v.to(E4M3)
            ckpt[key(k)], expanded[k] = (c if form == "float8" else c.to(torch.bfloat16)), c.to(torch.bfloat16)
        else:
            ckpt[key(k)], expanded[k] = v, v
    return ckpt, expanded


def _pair(family, form="float8", key=lambda k: k, **kw):
    """(FP8 model, bf16 model holding the expanded weights, FP8 checkpoint) with identical adapters."""
    src = tar._qwen(**kw) if family == "qwen" else tar._flux(**kw)
    base = {k.replace(".base_layer.", "."): v for k, v in src.state_dict().items() if ".lora_" not in k}
    ckpt, expanded = _fp8_checkpoint(base, form, key)
    lora = {k: v for k, v in src.state_dict().items() if ".lora_" in k}
    models = []
    for fw, sd in (("fp8", ckpt), ("bf16", expanded)):
        m = type(src)(src.config, device="cpu", _host_only=True, frozen_weights=fw)
        m.add_adapter(src.lora_rank, src.lora_rank * src.lora_scaling, target_modules=src.peft_config[src.adapter_name].target_modules)
        m.load_state_dict({**sd, **lora}, strict=True)
        models.append(m)
    return models[0], models[1], ckpt


# ------------------------------------------------------------------------------------------------------------------ format
def test_every_finite_code_round_trips_in_both_forms():
    from qflux_b200 import fp8
    codes = torch.tensor([c for c in range(256) if c & 0x7F != 0x7F], dtype=torch.uint8).view(E4M3)
    assert codes.numel() == 254
    up = codes.to(torch.bfloat16)
    assert up.view(torch.int16)[codes.view(torch.uint8) == 0x80].tolist() == [-32768]  # -0 stays -0 (0x8000)
    assert float(up[codes.view(torch.uint8) == 0x01]) == 2.0 ** -9  # the smallest subnormal
    for form in (codes, up):
        got = fp8.as_e4m3("w", form.view(2, 127))
        assert got.dtype == E4M3 and torch.equal(got.view(torch.uint8).reshape(-1), codes.view(torch.uint8))


@pytest.mark.parametrize("bad,what", [(0.3, "0.30"), (500.0, "500.0"), (float("inf"), "inf"), (float("nan"), "nan"),
                                      (2.0 ** -10, "0.0009765625")])
def test_a_bf16_value_that_is_not_e4m3_is_refused_by_name_and_value(bad, what):
    from qflux_b200 import fp8, lib
    w = torch.tensor([0.5, -0.0, 0.125] * 4, dtype=torch.bfloat16)
    w[7] = bad
    with pytest.raises(lib.QfxError, match=rf"`blk\.w`: element 7 = {what}"):
        fp8.as_e4m3("blk.w", w)


@pytest.mark.parametrize("code", [0x7F, 0xFF])
def test_nan_codes_and_other_dtypes_are_refused(code):
    from qflux_b200 import fp8, lib
    c = torch.zeros(32, dtype=torch.uint8)
    c[5] = code
    with pytest.raises(lib.QfxError, match=rf"`blk\.w`: element 5 is the float8-e4m3fn NaN code 0x{code:02x}"):
        fp8.as_e4m3("blk.w", c.view(E4M3))
    with pytest.raises(lib.QfxError, match="torch.float32"):
        fp8.as_e4m3("blk.w", torch.zeros(32))


def test_kernel_arguments_are_checked_before_any_cuda_call():
    from qflux_b200 import lib
    buf = torch.zeros(64, dtype=torch.uint8)
    p = buf.data_ptr() + (-buf.data_ptr()) % 16  # a 16-byte aligned address (never dereferenced: every call below is refused)
    for segs, n, msg in (([(p, p, 15)], 1, b"not a positive multiple of 16"), ([(0, p, 16)], 1, b"NULL pointer"),
                         ([(p + 8, p, 16)], 1, b"16-byte aligned"), ([(p, p + 2, 16)], 1, b"16-byte aligned"),
                         ([(p, p, 16)], 0, b"nseg=0"), ([(p, p, 16)] * 9, 9, b"nseg=9")):
        arr = (lib.Fp8Segment * len(segs))(*[lib.Fp8Segment(a, b, c) for a, b, c in segs])
        assert lib._lib.qfx_fp8_expand(arr, n, None) != 0
        assert msg in lib._lib.qfx_last_error()


@pytest.mark.parametrize("form", ["float8", "bf16"])
@pytest.mark.parametrize("prefix", ["", "base_layer", "transformer", "both"])
def test_fused_model_holds_the_expanded_weights(emu, form, prefix):
    def key(k):
        k = _base_layer(k) if prefix in ("base_layer", "both") else k
        return ("transformer." + k) if prefix in ("transformer", "both") else k
    m, ref, _ = _pair("qwen", form, key, L=2)
    assert m.frozen_weights == "fp8" and ref.frozen_weights == "bf16"
    views = ref._weight_views()
    for blk in range(m.L):  # every block matrix, expanded through the ring, equals the bf16 model's
        m._acquire(blk, -1)
        for k, v in m._weight_views(store=True).items():
            if k.startswith(f"transformer_blocks.{blk}.") and v.is_meta:
                kind = m._matrix_kind(k)
                got = m.w[kind][blk].reshape(-1)[v.storage_offset() - blk * m.w[kind].numel:][: v.numel()].view(v.shape)
                assert torch.equal(got, views[k]), k
        m._release(blk)
    for k, wk in (("img_in.weight", "img_in_w"), ("txt_in.weight", "txt_in_w"), ("proj_out.weight", "proj_out_w"),
                  ("norm_out.linear.weight", "norm_out_w"), ("transformer_blocks.1.attn.norm_q.weight", "qknorm_w")):
        t = m.w[wk] if wk != "qknorm_w" else m.w[wk][1, 0]
        assert torch.equal(t, views[k]) and t.dtype == torch.bfloat16, k  # outside the block matrices: bf16, upcast at load


def test_frozen_weight_bytes_are_the_computed_bytes(emu):
    m, _, _ = _pair("flux", nd=2, ns=3)
    D, L, Ls = m.D, m.L, m.Ls
    params = L * 2 * (6 + 3 + 1 + 4 + 4) * D * D + Ls * (3 + 3 + 4 + 5) * D * D
    assert sum(c.numel() * c.element_size() for c in m._fp8_store.values()) == params
    assert all(c.dtype == E4M3 for c in m._fp8_store.values())
    assert sum(r.gbuf.numel() * 2 for r in m._expand_rings) == 2 * 2 * (2 * 18 * D * D + 15 * D * D)
    assert not any(torch.is_tensor(m.w[k]) for k in m._fp8_store)  # the bf16 stacks were never allocated
    assert m._nf4_rings is None and not m._nf4_store


def test_a_bf16_model_upcasts_float8_tensors_as_before(emu):
    m, ref, ckpt = _pair("qwen", L=2)
    bf = type(m)(m.config, device="cpu", _host_only=True)
    bf.load_state_dict(ckpt, strict=True)
    for k, v in ref._weight_views().items():
        assert torch.equal(bf._weight_views()[k], v), k


# ------------------------------------------------------------------------------------------------------------------ parity
@pytest.mark.parametrize("kind", ["dense", "plus", "multi"])
def test_qwen_fp8_equals_bf16_with_expanded_weights(emu, kind):
    m, ref, _ = _pair("qwen", "bf16", targets=QWEN_TARGETS)
    batch = tar._qwen_batch(kind)
    tar._same(tar._fused(m, "qwen", batch), tar._fused(ref, "qwen", batch))


@pytest.mark.parametrize("kind", ["dense", "multi"])
def test_flux_fp8_equals_bf16_with_yaml_targets(emu, kind):
    m, ref, _ = _pair("flux")
    assert any(k.startswith("single_") for k in m.mod_sites.get("sgl", {}).get("names", [])) and any(s[0] == -1 for s in m.sites)
    batch = tar._flux_batch(kind)
    tar._same(tar._fused(m, "flux", batch), tar._fused(ref, "flux", batch))


@pytest.mark.parametrize("family", ["qwen", "flux"])
@pytest.mark.parametrize("mode", ["partial", "all"])
def test_fp8_with_forced_recompute(emu, monkeypatch, family, mode):
    from qflux_b200 import mmdit_base
    monkeypatch.setattr(mmdit_base, "plan_activation_memory", tar.force_plan(mode))
    m, ref, _ = _pair(family)
    batch = (tar._qwen_batch if family == "qwen" else tar._flux_batch)("dense")
    tar._same(tar._fused(m, family, batch), tar._fused(ref, family, batch))
    assert m.activation_plan.recompute


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
def test_fp8_gradient_accumulation_and_autograd_bridges(emu, family):
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
        step.compute_loss(emb, noise, u).backward()  # step bridge
        g1 = [p.grad.clone() for p in model.parameters()]
        model.zero_grad()
        pred = _model_bridge_pred(model, family, mk("dense", 3))
        pred.float().square().mean().backward()  # model bridge (ModelFn)
        g2 = [p.grad.clone() for p in model.parameters()]
        res.append((gacc, g1, g2, pred.detach()))
    assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][3], res[1][3])
    for a, b in zip(res[0][1] + res[0][2], res[1][1] + res[1][2]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("family", ["qwen", "flux"])
def test_fp8_no_grad_forward_and_sampler(emu, family):
    m, ref, _ = _pair(family)
    mk = tar._qwen_batch if family == "qwen" else tar._flux_batch
    with torch.no_grad():
        assert torch.equal(_model_bridge_pred(m, family, mk("dense", 4)), _model_bridge_pred(ref, family, mk("dense", 4)))
    if family == "qwen":
        from qflux_b200.sampler import sample_qwen
        emb, noise, _ = mk("dense", 5)
        emb = dict(emb, latents=noise, prompt_embeds_mask=torch.ones(emb["prompt_embeds"].shape[:2], dtype=torch.int64),
                   num_inference_steps=2)
        assert torch.equal(sample_qwen(m, emb), sample_qwen(ref, emb))


# ------------------------------------------------------------------------------------------------------------------ integration
def _upcast_reference(ckpt, cfg, peft=None):
    """A reference-like transformer holding what `from_pretrained(fp8 checkpoint, torch_dtype=bf16)` holds: the bf16 upcast
    weights, optionally under a PEFT adapter (`.base_layer.` names plus the LoRA factors)."""
    class Ref(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.config = cfg
            if peft is not None:
                self.peft_config = {"default": peft}

        def state_dict(self, *a, **k):
            return dict(ckpt)
    return Ref()


@pytest.mark.parametrize("family", ["qwen", "flux"])
def test_from_reference_and_patch_trainer_on_an_upcast_fp8_reference(emu, family):
    from qflux_b200 import integration
    m, ref, _ = _pair(family, "bf16")
    src = {k: v for k, v in m.state_dict().items() if ".lora_" in k}
    _, expanded = _fp8_checkpoint({k.replace(".base_layer.", "."): v for k, v in ref.state_dict().items() if ".lora_" not in k})
    lora_mods = {k.rsplit(".lora_", 1)[0] for k in src}
    ckpt = {(k[: -len(".weight")] + ".base_layer.weight" if k.endswith(".weight") and k[: -len(".weight")] in lora_mods else k): v
            for k, v in expanded.items()}
    ckpt.update(src)
    cfg = {k: getattr(m.config, k) for k in m.config.__dataclass_fields__}
    pc = m.peft_config[m.adapter_name]
    dit = integration.from_reference(_upcast_reference(ckpt, cfg, pc), _host_only=True, frozen_weights="fp8")
    assert dit.frozen_weights == "fp8"
    batch = (tar._qwen_batch if family == "qwen" else tar._flux_batch)("dense")
    tar._same(tar._fused(dit, family, batch), tar._fused(ref, family, batch))
    # the trainer's config names an FP8 checkpoint: patch_trainer keeps the block weights FP8-resident; otherwise today's bf16 path
    for qt, want in (("pretrain_fp8", "fp8"), ("pretrain_fp16", "bf16"), (None, "bf16")):
        trainer = type("T", (), {})()
        trainer.dit = _upcast_reference(ckpt, cfg, pc)
        if qt is not None:
            trainer.config = type("Cfg", (), {"quantization_type": qt, "train": None})()
        integration.patch_trainer(trainer, _host_only=True)
        assert trainer.dit.frozen_weights == want, qt
        if want == "fp8":
            tar._same(tar._fused(trainer.dit, family, batch), tar._fused(ref, family, batch))


def test_save_and_reload_the_lora_of_an_fp8_model(emu):
    m, _, ckpt = _pair("qwen")
    sd = m.state_dict()
    assert not any(k.startswith("transformer_blocks.") and ".lora_" not in k for k in sd)  # LoRA and the non-block tensors only
    assert "img_in.weight" in sd and sd["img_in.weight"].dtype == torch.bfloat16
    lora = {"transformer." + k.replace(".default", ""): v for k, v in sd.items() if ".lora_" in k}
    fresh = type(m)(m.config, device="cpu", _host_only=True, frozen_weights="fp8")
    fresh.load_state_dict(ckpt, strict=False)
    fresh.load_lora_adapter(lora)
    assert all(torch.equal(fresh._lora_params[k], p) for k, p in m._lora_params.items())


# ------------------------------------------------------------------------------------------------------------------ refusals
def test_refuses_sharding_and_merge_adapter(emu):
    from qflux_b200 import lib
    m, _, _ = _pair("qwen", L=2)
    with pytest.raises(lib.QfxError, match="sharded FP8"):
        m.shard_frozen_weights()
    with pytest.raises(lib.QfxError, match="FP8-resident"):
        m.merge_adapter()


def test_refuses_mixed_formats_a_bf16_checkpoint_nan_codes_and_nf4(emu):
    import nf4_ref
    from qflux_b200 import lib
    m, ref, ckpt = _pair("qwen", L=2)
    new = lambda: type(m)(m.config, device="cpu", _host_only=True, frozen_weights="fp8")
    # a stacked kind whose layers arrive in mixed forms (block 0 float8, block 1 its bf16 upcast)
    mixed = {k: (v.to(torch.bfloat16) if k.startswith("transformer_blocks.1.") and v.dtype == E4M3 else v) for k, v in ckpt.items()}
    with pytest.raises(lib.QfxError, match=r"transformer_blocks\.1\..* arrives as torch.bfloat16, .* arrived as "
                                           r"torch.float8_e4m3fn: the layers of a stacked kind must arrive in one format"):
        new().load_state_dict(mixed)
    # a genuine bf16 checkpoint: named by its first block matrix that is not an e4m3 value
    base = {k.replace(".base_layer.", "."): v for k, v in ref.state_dict().items() if ".lora_" not in k}
    genuine = {k: (v * 1.01 if k.endswith(".weight") and v.ndim == 2 else v) for k, v in base.items()}
    first = next(k for k in genuine if k.startswith("transformer_blocks.") and genuine[k].ndim == 2)
    with pytest.raises(lib.QfxError, match=rf"`{first}`: element \d+ = .* is not a float8-e4m3fn value"):
        new().load_state_dict(genuine)
    nan = dict(ckpt)
    k = "transformer_blocks.1.attn.to_k.weight"
    raw = nan[k].view(torch.uint8).clone()
    raw[3, 9] = 0xFF
    nan[k] = raw.view(E4M3)
    with pytest.raises(lib.QfxError, match=rf"`{k}`: element {3 * raw.shape[1] + 9} is the float8-e4m3fn NaN code 0xff"):
        new().load_state_dict(nan)
    nf4 = nf4_ref.to_nf4_state_dict(base, _in_blocks)
    with pytest.raises(lib.QfxError, match="NF4 weight, but this model keeps its block matrices FP8-resident"):
        new().load_state_dict(nf4)
    with pytest.raises(lib.QfxError, match="'fp8'"):
        type(m)(m.config, device="cpu", _host_only=True, frozen_weights="fp16")


# ------------------------------------------------------------------------------------------------------------------ GPU
def _gpu_case(name):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "fp8_check.py"), name], capture_output=True, text=True, cwd=ROOT)
    print(r.stdout[-4000:], r.stderr[-4000:])
    assert r.returncode == 0, name


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["kernel_all_codes", "kernel_qwen_double", "kernel_flux_single", "qwen_step_parity",
                                  "flux_step_parity", "graph_replay", "infer_replay"])
def test_gpu(name):
    _gpu_case(name)
