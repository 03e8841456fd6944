"""Row (b) of SURVEY.md §8 — the drop-in boundary — exercised with the REFERENCE'S OWN trainer code (tests that take the `ref` fixture
need the reference checkout at /root/reference and skip without it; `diffusers` / `peft` / `accelerate` come from tests/shims).  What
the reference computes as plain data — RoPE tables, sampling schedules, a cache directory it wrote — is stored in
tests/golden/boundary_golden.pt (tests/golden/make_boundary_golden.py), so those comparisons run everywhere.  The fused model runs on
CPU with emulated kernels (tests/emu_lib.py): what is under test is the interface, not the arithmetic.

Driven reference code: `BaseTrainer.add_lora_adapter`, `.load_pretrain_lora_model`, `.save_lora`, `.clip_gradients`, `.forward_loss`,
`QwenImageEditTrainer._compute_loss`, `utils.lora_utils.get_lora_layers / classify_lora_weight`, `QwenEmbedRope`,
the loop body of `train_epoch` (base_trainer.py:518-533)."""
import os
import sys
import types

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF_SRC = "/root/reference/src"

sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, os.path.join(HERE, "shims"))


@pytest.fixture(scope="module")
def ref():
    if not os.path.isdir(os.path.join(REF_SRC, "qflux")):
        pytest.skip("runs the reference's trainer code: needs the reference checkout at /root/reference")
    import stub_importer
    stub_importer.install()
    if REF_SRC not in sys.path:
        sys.path.insert(0, REF_SRC)
    import make_ref_model_golden as mg
    return mg


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(HERE, "golden", "boundary_golden.pt"), weights_only=False)


@pytest.fixture()
def emu():
    import emu_lib
    from qflux_b200 import lib
    restore = emu_lib.install(lib)
    yield
    restore()


def _cfg(r=4, alpha=8, targets=("to_q", "to_k", "to_v", "to_out.0"), pretrained=None):
    lora = types.SimpleNamespace(r=r, lora_alpha=alpha, init_lora_weights="gaussian", target_modules=list(targets), pretrained_weight=pretrained)
    return types.SimpleNamespace(model=types.SimpleNamespace(lora=lora), train=types.SimpleNamespace(max_grad_norm=0.5, gradient_accumulation_steps=1))


def _fused(host_only=True):
    import ref_common as rc
    from qflux_b200.qwen_model import QwenB200Config, QwenImageB200
    c = rc.QWEN_HD128
    return QwenImageB200(QwenB200Config(num_layers=c["num_layers"], num_attention_heads=c["num_attention_heads"],
                                        joint_attention_dim=c["joint_attention_dim"]), device="cpu", _host_only=host_only)


def test_reference_add_lora_adapter_and_module_scan(ref, emu):
    """base_trainer.py:929-941 on the fused model: LoraConfig object + adapter_name; get_lora_layers (lora_utils.py:25-38) finds child
    modules whose parameters are exactly the trainable LoRA parameters (what accelerator_prepare wraps / FSDP ignores)."""
    from qflux.trainer.base_trainer import BaseTrainer
    from qflux.utils.lora_utils import get_lora_layers
    m = _fused()
    BaseTrainer.add_lora_adapter(m, _cfg(), "lora_edit")
    names = [n for n, _ in m.named_parameters()]
    assert len(names) == 2 * 4 * 2 and all(".lora_A.lora_edit.weight" in n or ".lora_B.lora_edit.weight" in n for n in names)
    assert all(p.requires_grad for p in m.parameters()) and all("lora" in n for n in names)  # qwen_image_edit_trainer.py:314-318
    assert set(m.peft_config) == {"lora_edit"} and m.peft_config["lora_edit"].r == 4
    layers = get_lora_layers(m)
    assert layers and all(isinstance(v, torch.nn.Module) for v in layers.values())
    found = {id(p) for v in layers.values() for p in v.parameters()}
    assert found == {id(p) for p in m.parameters()}
    with pytest.raises(Exception):
        m.set_adapter("other")
    m.set_adapter("lora_edit")
    assert m.to("cpu") is m and m.to(torch.bfloat16) is m  # no-op moves are accepted (base_trainer.py:388) ...
    with pytest.raises(Exception):
        m.to(torch.float32)                                  # ... re-typing the fused HBM layout is refused loudly


def test_pos_embed_matches_reference_rope(golden):
    """`dit.pos_embed([shapes], [T], device)` (qwen_image_edit_trainer.py:734) vs the reference's QwenEmbedRope (scale_rope=True)."""
    m = _fused()
    for c in golden["rope"]:
        a_v, a_t = m.pos_embed([c["shapes"]], [c["T"]], device=torch.device("cpu"))
        b_v, b_t = c["vid"], c["txt"]
        assert a_v.shape == b_v.shape and a_t.shape == b_t.shape
        assert (a_v - b_v).abs().max() < 2e-5 and (a_t - b_t).abs().max() < 2e-5


def test_patch_trainer_runs_the_reference_loop_body(ref, emu):
    """patch_trainer on a reference trainer object: the reference's own loop body (training_step -> accelerator.backward -> clip_gradients
    -> optimizer.step -> zero_grad) runs unmodified on the fused model and tracks the un-patched reference run."""
    import ref_common as rc
    from accelerate import Accelerator
    from qflux.losses import MseLoss
    from qflux.trainer.qwen_image_edit_trainer import QwenImageEditTrainer
    import qflux.trainer.qwen_image_edit_trainer as qt
    from qflux_b200 import patch_trainer
    from qflux_b200.mmdit_base import FusedMMDiTBase
    spec = rc.CASES["qwen_hd128"]
    x = rc.rand_inputs(spec)
    emb = {k: v for k, v in x.items() if k != "u"}
    orig = qt.compute_density_for_timestep_sampling
    qt.compute_density_for_timestep_sampling = lambda **kw: x["u"].clone()
    try:
        results = {}
        for which in ("reference", "b200"):
            dit, _ = ref.build_reference(spec)
            tr = ref._trainer(QwenImageEditTrainer, dit, MseLoss(reduction="mean"))
            tr.config = _cfg()
            tr.adapter_name = "default"
            if which == "b200":
                patch_trainer(tr, _host_only=True)
                assert isinstance(tr.dit, FusedMMDiTBase) and tr.dit.peft_config["default"].r == 4
            tr.optimizer = torch.optim.AdamW([p for p in tr.dit.parameters() if p.requires_grad], lr=1e-2, weight_decay=0.0)
            losses = []
            for it in range(3):  # base_trainer.py:518-533
                with tr.accelerator.accumulate(tr.dit):
                    torch.manual_seed(100 + it)
                    e = dict(emb)
                    if which == "b200":  # the reference draws randn_like(image_latents) in fp32 on the CPU: hand the fused step the same draw
                        e["noise"] = torch.randn_like(emb["image_latents"])
                        e["u"] = x["u"]
                    loss = tr._compute_loss(e)
                    tr.accelerator.backward(loss)
                    tr.clip_gradients()
                    tr.optimizer.step()
                    tr.optimizer.zero_grad()
                losses.append(float(loss))
            results[which] = (losses, {n: p.detach().float().clone() for n, p in tr.dit.named_parameters() if p.requires_grad}, tr)
    finally:
        qt.compute_density_for_timestep_sampling = orig
    (l_r, p_r, _), (l_b, p_b, tr_b) = results["reference"], results["b200"]
    assert all(abs(a - b) < 2e-2 for a, b in zip(l_r, l_b)), (l_r, l_b)
    assert l_b[-1] < l_b[0]  # the optimizer actually moved the LoRA parameters in the right direction
    assert set(p_r) == set(p_b)
    num = sum(((p_b[n] - p_r[n]) ** 2).sum() for n in p_r)
    den = sum((p_r[n] ** 2).sum() for n in p_r)
    assert float((num / den).sqrt()) < 2e-2  # bf16 parameters vs the fp32 reference run after three AdamW steps


def test_save_lora_roundtrip_through_reference_code(ref, emu, tmp_path):
    """save_lora (base_trainer.py:858-875: unwrap -> get_peft_model_state_dict -> convert_state_dict_to_diffusers ->
    pipeline.save_lora_weights -> safetensors) on the fused model; the file loads back into the fused model AND into the reference model
    (`load_lora_adapter`, :983), and `load_pretrain_lora_model` (:943-1002) resumes from it."""
    import ref_common as rc
    import safetensors.torch
    from accelerate import Accelerator
    from diffusers import FluxKontextPipeline
    from qflux.models.transformer_qwenimage import QwenImageTransformer2DModel
    from qflux.trainer.base_trainer import BaseTrainer
    from qflux.trainer.qwen_image_edit_trainer import QwenImageEditTrainer
    from qflux.utils.lora_utils import classify_lora_weight
    m = _fused()
    BaseTrainer.add_lora_adapter(m, _cfg(), "default")
    rc.det_fill_(type("B", (), {"named_parameters": lambda s: iter(m._lora_params.items())})(), 5)
    tr = object.__new__(QwenImageEditTrainer)
    tr.accelerator, tr.dit, tr.adapter_name, tr.pipeline_class = Accelerator(), m, "default", FluxKontextPipeline
    folder = str(tmp_path / "ckpt")
    tr.save_lora(folder)
    path = os.path.join(folder, "pytorch_lora_weights.safetensors")
    sd = safetensors.torch.load_file(path)
    assert len(sd) == 16 and all(k.startswith("transformer.") and (k.endswith(".lora_A.weight") or k.endswith(".lora_B.weight")) for k in sd)
    assert classify_lora_weight(path) == "PEFT"
    want = {n: p.detach().clone() for n, p in m.named_parameters()}
    # (1) into a fresh fused model through the diffusers entry point
    m2 = _fused()
    m2.load_lora_adapter(path, adapter_name="default")
    assert m2.lora_rank == 4 and all(torch.equal(p, want[n]) for n, p in m2.named_parameters())
    # (2) into the reference model through ITS load_lora_adapter
    refm = QwenImageTransformer2DModel(**rc.QWEN_HD128)
    refm.load_lora_adapter(path, adapter_name="default")
    got = {n: p for n, p in refm.named_parameters() if "lora_" in n}
    assert set(got) == set(want) and all(torch.equal(got[n].to(torch.bfloat16), want[n]) for n in want)
    # (3) the trainer's resume path: classify -> add_lora_adapter -> load_state_dict(strict=False) -> no unexpected keys
    m3 = _fused()
    BaseTrainer.load_pretrain_lora_model(m3, _cfg(pretrained=path), "default")
    assert all(torch.equal(p, want[n]) for n, p in m3.named_parameters())
    # state_dict() hands out compact tensors (safetensors refuses views), torch.save stays small
    assert all(v.is_contiguous() for v in m.state_dict().values() if v.ndim == 2 and v.shape[1] == 4)


def test_fused_adamw_honours_the_optimizer_contract(emu):
    """ADVICE r1: `step(closure=None)` positional contract, AcceleratedOptimizer-style wrappers (`.optimizer`), mean over ranks x micro-steps."""
    import ref_common as rc
    from qflux_b200.optim import FusedLoraAdamW
    from qflux_b200.train_step import QwenImageEditStep, _sync_and_step
    sys.path.insert(0, HERE)
    from test_reference_goldens import _b200_model
    m, _ = _b200_model(rc.CASES["qwen_hd128"], "cpu", True)  # name-derived non-zero weights (an all-zero model has zero LoRA gradients)
    opt = FusedLoraAdamW(m, lr=1e-2)

    class Wrapped:  # accelerate.optimizer.AcceleratedOptimizer: forwards step(closure) to .optimizer
        def __init__(self, o):
            self.optimizer = o

        def step(self, closure=None):
            return self.optimizer.step(closure)
    x = rc.rand_inputs(rc.CASES["qwen_hd128"])
    emb = {k: x[k] for k in ("image_latents", "control_latents", "prompt_embeds", "img_shapes")}
    step = QwenImageEditStep(m, "mse", max_grad_norm=1.0)
    before = [p.detach().clone() for p in m.parameters()]
    step.train_step(emb, Wrapped(opt), noise=torch.randn(2, 16, 64).bfloat16(), u=x["u"])
    assert opt.step_count == 1 and any(not torch.equal(a, b) for a, b in zip(before, m.parameters()))
    assert opt.step(None) is None and opt.step_count == 2          # positional closure slot accepts None
    assert opt.step(lambda: torch.tensor(3.0)).item() == 3.0        # and a real closure
    # the divisor set by the sync (world x micro-steps) is what a later plain step() uses: a summed gradient is never applied as-is
    m.G32.fill_(2.0)
    _sync_and_step(m, opt, 0.0, micro_steps=4)
    assert opt.grad_divisor == 4 and abs(float(opt.grad_norm_sq.sqrt()) - 0.5 * m.G32.numel() ** 0.5) < 1e-2 * m.G32.numel() ** 0.5


def test_patch_trainer_flux_shared_and_multires(ref, emu):
    """patch_trainer on the FLUX-Kontext trainer: the reference's `embeddings` dict (pixel `image`, pixel-space `img_shapes`, `control_ids`)
    goes through the fused step unchanged, in shared mode (flux_kontext_trainer.py:494-577) and in multi-resolution mode (:579-796)."""
    import ref_common as rc
    from qflux.losses import AttentionMaskMseLoss, MseLoss
    from qflux.trainer.flux_kontext_trainer import FluxKontextLoraTrainer
    from qflux_b200 import patch_trainer
    for case, crit in (("flux_hd128", MseLoss(reduction="mean")), ("flux_custom_multires", AttentionMaskMseLoss(reduction="mean"))):
        spec = rc.CASES[case]
        x = rc.rand_inputs(spec)
        emb = {k: v for k, v in x.items() if k not in ("img_shapes_latent", "hw")}
        if spec["kind"] == "flux":
            h_, w_ = x["hw"]
            emb["control_ids"] = FluxKontextLoraTrainer._prepare_latent_image_ids(1, h_, w_, torch.device("cpu"), torch.float32)
            emb["control_ids"][..., 0] = 1
            emb["img_shapes"] = [[(3, h_ * 16, w_ * 16), (3, h_ * 16, w_ * 16)]] * spec["B"]
        else:
            emb["timestep"] = x["timestep"].view(-1, 1)
        out = {}
        for which in ("reference", "b200"):
            dit, _ = ref.build_reference(spec)
            tr = ref._trainer(FluxKontextLoraTrainer, dit, crit)
            tr.config = _cfg()
            e = dict(emb)
            if which == "b200":
                patch_trainer(tr, _host_only=True)
                if spec["kind"] == "flux_multi":  # the fused step takes one padded noise tensor and a flat timestep vector
                    lt = [s[0][1] * s[0][2] for s in x["img_shapes_latent"]]
                    nz = torch.zeros(len(lt), max(lt), 64)
                    for b, n in enumerate(lt):
                        nz[b, :n] = x["noise"][b]
                    e["noise"], e["timestep"] = nz, x["timestep"]
            loss = tr._compute_loss(e)
            loss.backward()
            out[which] = (float(loss), {n: p.grad.float().clone() for n, p in tr.dit.named_parameters() if p.requires_grad and p.grad is not None})
        (l_r, g_r), (l_b, g_b) = out["reference"], out["b200"]
        assert abs(l_r - l_b) < 1e-2, (case, l_r, l_b)
        num = sum(((g_b[n] - g_r[n]) ** 2).sum() for n in g_r)
        den = sum((g_r[n] ** 2).sum() for n in g_r)
        assert set(g_r) <= set(g_b) and float((num / den).sqrt()) < 2e-2, case


def test_sampler_schedule_matches_reference_prepare_predict_timesteps(golden):
    """§8 f2: `flow_match_sigmas` vs the reference's `BaseTrainer.prepare_predict_timesteps` (base_trainer.py:1009-1043 -> calculate_shift,
    retrieve_timesteps -> FlowMatchEulerDiscreteScheduler.set_timesteps(sigmas=, mu=)), for the Qwen-Image and the FLUX scheduler configs,
    and the Euler update vs `scheduler.step`."""
    from qflux_b200.sampler import _euler_step, calculate_shift, flow_match_sigmas
    assert {c["config"] for c in golden["schedules"]} == {"qwen", "flux"} and len(golden["schedules"]) == 6
    for c in golden["schedules"]:
        conf, steps, seq, ts = c["conf"], c["steps"], c["seq"], c["timesteps"]
        assert abs(calculate_shift(seq, conf["base_image_seq_len"], conf["max_image_seq_len"], conf["base_shift"], conf["max_shift"])
                   - c["shift"]) < 1e-12
        sig = flow_match_sigmas(steps, seq, base_seq_len=conf["base_image_seq_len"], max_seq_len=conf["max_image_seq_len"],
                                base_shift=conf["base_shift"], max_shift=conf["max_shift"], shift_terminal=conf.get("shift_terminal"))
        assert c["n"] == steps and sig.numel() == steps + 1 and sig[-1] == 0
        assert torch.allclose(sig[:-1] * 1000, ts, rtol=2e-6, atol=1e-4), (c["config"], steps, seq)
        assert torch.allclose(sig, c["sigmas"], rtol=2e-6, atol=1e-7)
        # one Euler step of the loop in sampler.py == scheduler.step (fp32 update, model dtype out)
        assert torch.equal(c["euler"], _euler_step(c["x"], c["v"], sig, 0))


def test_loader_reads_a_cache_written_by_the_reference(golden, tmp_path):
    """f3: the cache directory was produced by the reference's own `EmbeddingCacheManager.save_cache_embedding` (data/cache_manager.py:
    46-93); `CachedEmbeddingLoader` must read back what the reference's `load_cache` + `pad_to_max_shape` (utils/tools.py:399-425) read
    from it, sample by sample (values, fp16 storage, pixel `img_shapes` converted to latent-patch units, pad-to-max collate)."""
    from qflux_b200.cache_loader import CachedEmbeddingLoader
    c = golden["cache"]
    for rel, data in c["files"].items():
        p = tmp_path / rel
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_bytes(data)
    ours = list(CachedEmbeddingLoader(str(tmp_path), batch_size=3, device="cpu", shuffle=False, drop_last=False))
    assert len(ours) == 1
    b = ours[0]
    for key, want in c["want"].items():
        assert b[key].dtype == torch.float16 and torch.equal(b[key], want), key
    assert b["img_shapes"] == [[(1, H // 16, W // 16)] * 2 for H, W in c["sizes"]]
    assert b["prompt_embeds_mask"].sum(1).tolist() == [6, 11, 16]
    # ... and the same batch again from the packed shards written off that cache
    from qflux_b200.cache_loader import pack_cache
    pack_cache(str(tmp_path))
    p = list(CachedEmbeddingLoader(str(tmp_path), batch_size=3, device="cpu", shuffle=False, drop_last=False, packed=True))[0]
    assert all(torch.equal(p[k], b[k]) for k in ("image_latents", "control_latents", "prompt_embeds", "prompt_embeds_mask")) and p["img_shapes"] == b["img_shapes"]


def test_dreamomni2_trainer_rides_the_flux_kontext_path(ref):
    """§8 f4: the reference's DreamOmni2 trainer only changes what happens BEFORE the embeddings exist (VLM prompt optimisation); its loss
    recipes are FluxKontextLoraTrainer's own, i.e. exactly what FluxKontextStep / patch_trainer replace."""
    from qflux.trainer.dreamomni2_trainer import DreamOmni2Trainer
    from qflux.trainer.flux_kontext_trainer import FluxKontextLoraTrainer
    assert issubclass(DreamOmni2Trainer, FluxKontextLoraTrainer)
    for name in ("_compute_loss", "_compute_loss_shared_mode", "_compute_loss_multi_resolution_mode"):
        assert getattr(DreamOmni2Trainer, name) is getattr(FluxKontextLoraTrainer, name), name
    # likewise BASELINE config 4's trainer: Edit-Plus only changes how the (several) control images are encoded and concatenated
    from qflux.trainer.qwen_image_edit_plus_trainer import QwenImageEditPlusTrainer
    from qflux.trainer.qwen_image_edit_trainer import QwenImageEditTrainer
    assert issubclass(QwenImageEditPlusTrainer, QwenImageEditTrainer) and QwenImageEditPlusTrainer._compute_loss is QwenImageEditTrainer._compute_loss


def test_reference_validation_loop_runs_on_the_fused_model(ref, emu):
    """§8 f2 pinned to the reference's own loop: `QwenImageEditTrainer.sampling_from_embeddings` (qwen_image_edit_trainer.py:1116-1289 —
    shifted schedule, `dit.cache_context`, true CFG with norm rescale, `scheduler.step`) is run UNMODIFIED with `self.dit` = the fused
    model and must produce the latents of `qflux_b200.sampler.sample_qwen` on the same model, and — within bf16 tolerance — those of the
    same loop driving the reference's own transformer."""
    import contextlib
    import io
    import ref_common as rc
    from diffusers.schedulers.scheduling_flow_match_euler_discrete import FlowMatchEulerDiscreteScheduler
    from qflux.trainer.base_trainer import BaseTrainer
    from qflux.trainer.qwen_image_edit_trainer import QwenImageEditTrainer
    from qflux_b200 import from_reference
    from qflux_b200.sampler import sample_qwen
    spec = rc.CASES["qwen_hd128"]
    ref_dit, _ = ref.build_reference(spec)
    fused = from_reference(ref_dit, _host_only=True)
    x = rc.rand_inputs(spec)
    B, L = x["image_latents"].shape[:2]
    T = x["prompt_embeds"].shape[1]
    g = torch.Generator().manual_seed(77)
    sched = dict(num_train_timesteps=1000, shift=1.0, use_dynamic_shifting=True, base_shift=0.5, max_shift=0.9, base_image_seq_len=256,
                 max_image_seq_len=8192, shift_terminal=0.02)
    emb = dict(num_inference_steps=4, true_cfg_scale=3.0, guidance=1.0, height=512, width=512, negative_prompt="bad",
               control_latents=x["control_latents"].bfloat16(), prompt_embeds=x["prompt_embeds"].bfloat16(),
               prompt_embeds_mask=torch.ones(B, T, dtype=torch.int64), img_shapes=x["img_shapes"],
               negative_prompt_embeds=(torch.randn(B, T - 3, x["prompt_embeds"].shape[2], generator=g) * 3).bfloat16(),
               negative_prompt_embeds_mask=torch.ones(B, T - 3, dtype=torch.int64), latents=torch.randn(B, L, 64, generator=g).bfloat16())

    def reference_loop(dit, dtype):
        tr = types.SimpleNamespace(dit=dit, vae_scale_factor=8, weight_dtype=dtype, scheduler=None,
                                   sampling_scheduler=FlowMatchEulerDiscreteScheduler(**sched))
        tr.prepare_predict_timesteps = lambda *a, **k: BaseTrainer.prepare_predict_timesteps(tr, *a, **k)
        with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
            return QwenImageEditTrainer.sampling_from_embeddings(tr, dict(emb))
    via_reference_loop = reference_loop(fused, torch.bfloat16)
    ours = sample_qwen(fused, dict(emb), scheduler_kwargs=dict(base_seq_len=256, max_seq_len=8192, base_shift=0.5, max_shift=0.9, shift_terminal=0.02))
    assert via_reference_loop.shape == ours.shape == (B, L, 64)
    assert ((via_reference_loop.float() - ours.float()).norm() / ours.float().norm()).item() < 2e-3, "sampler.py must be the reference's loop"
    want = reference_loop(ref_dit.float(), torch.float32)  # the reference's loop on the reference's own fp32 transformer
    assert ((ours.float() - want).norm() / want.norm()).item() < 3e-2


def test_merge_adapter_like_peft(ref, emu):
    """`BaseTrainer.merge_lora` -> `dit.merge_adapter()` (base_trainer.py:413-416): after merging, the adapter-free forward of the
    merged weights equals the adapted forward; `unmerge_adapter()` brings the factors back."""
    import ref_common as rc
    from qflux.trainer.base_trainer import BaseTrainer
    from qflux_b200 import from_reference
    spec = rc.CASES["qwen_hd128"]
    ref_dit, _ = ref.build_reference(spec)
    m = from_reference(ref_dit, _host_only=True)
    x = rc.rand_inputs(spec)
    packed = torch.cat([x["image_latents"], x["control_latents"]], 1).bfloat16()
    kw = dict(hidden_states=packed, timestep=torch.tensor([0.5] * packed.shape[0]), encoder_hidden_states=x["prompt_embeds"].bfloat16(),
              encoder_hidden_states_mask=torch.ones(packed.shape[0], x["prompt_embeds"].shape[1], dtype=torch.int64), img_shapes=x["img_shapes"])
    with torch.no_grad():
        before = m(**kw)[0].float()
        B_norm = sum(float(p.float().norm()) for k, p in m._lora_params.items() if ".lora_B." in k)
        BaseTrainer.merge_lora(types.SimpleNamespace(dit=m))
        assert all(float(p.abs().max()) == 0 for k, p in m._lora_params.items() if ".lora_B." in k) and B_norm > 0
        merged = m(**kw)[0].float()
        m.unmerge_adapter()
        after = m(**kw)[0].float()
    assert ((merged - before).norm() / before.norm()).item() < 1e-2
    assert ((after - before).norm() / before.norm()).item() < 1e-2
    assert abs(sum(float(p.float().norm()) for k, p in m._lora_params.items() if ".lora_B." in k) - B_norm) < 1e-6


def test_reference_flux_validation_loop_runs_on_the_fused_model(ref, emu):
    """The FLUX-Kontext counterpart: `FluxKontextLoraTrainer.sampling_from_embeddings` (flux_kontext_trainer.py:902-976; plain CFG, no norm
    rescale) unmodified on the fused FLUX model vs `sample_flux`, and vs the same loop on the reference's own transformer."""
    import contextlib
    import io
    import ref_common as rc
    from diffusers.schedulers.scheduling_flow_match_euler_discrete import FlowMatchEulerDiscreteScheduler
    from qflux.trainer.base_trainer import BaseTrainer
    from qflux.trainer.flux_kontext_trainer import FluxKontextLoraTrainer
    from qflux_b200 import from_reference
    from qflux_b200.sampler import sample_flux
    from qflux_b200.train_step import FluxKontextStep
    spec = rc.CASES["flux_hd128"]
    ref_dit, _ = ref.build_reference(spec)
    fused = from_reference(ref_dit, _host_only=True)
    x = rc.rand_inputs(spec)
    B, L = x["image_latents"].shape[:2]
    T, J = x["prompt_embeds"].shape[1:]
    hw = int(L ** 0.5)
    g = torch.Generator().manual_seed(78)
    sched = dict(num_train_timesteps=1000, shift=3.0, use_dynamic_shifting=True, base_shift=0.5, max_shift=1.15, base_image_seq_len=256,
                 max_image_seq_len=4096)
    emb = dict(num_inference_steps=4, true_cfg_scale=2.5, guidance=3.5, control_latents=x["control_latents"].bfloat16(),
               control_ids=FluxKontextStep.latent_image_ids(hw, hw, "cpu", 1.0), latent_ids=FluxKontextStep.latent_image_ids(hw, hw, "cpu", 0.0),
               latents=torch.randn(B, L, 64, generator=g).bfloat16(), pooled_prompt_embeds=x["pooled_prompt_embeds"].bfloat16(),
               prompt_embeds=x["prompt_embeds"].bfloat16(), text_ids=torch.zeros(T, 3),
               negative_pooled_prompt_embeds=torch.randn(B, x["pooled_prompt_embeds"].shape[1], generator=g).bfloat16(),
               negative_prompt_embeds=torch.randn(B, T, J, generator=g).bfloat16(), negative_text_ids=torch.zeros(T, 3))

    def reference_loop(dit, dtype):
        tr = types.SimpleNamespace(dit=dit, weight_dtype=dtype, scheduler=None, sampling_scheduler=FlowMatchEulerDiscreteScheduler(**sched))
        tr.prepare_predict_timesteps = lambda *a, **k: BaseTrainer.prepare_predict_timesteps(tr, *a, **k)
        with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()):
            return FluxKontextLoraTrainer.sampling_from_embeddings(tr, dict(emb))
    via_reference_loop = reference_loop(fused, torch.bfloat16)
    ours = sample_flux(fused, dict(emb), scheduler_kwargs=dict(base_seq_len=256, max_seq_len=4096, base_shift=0.5, max_shift=1.15))
    assert via_reference_loop.shape == ours.shape == (B, L, 64)
    assert ((via_reference_loop.float() - ours.float()).norm() / ours.float().norm()).item() < 2e-3, "sampler.py must be the reference's loop"
    # against the reference's own transformer in bf16 (an fp32 run is not comparable over several steps: a bf16 FLUX model multiplies the
    # timestep by 1000 IN bf16, transformer_flux.py:707-710, so its time embedding differs from the fp32 model's at most sigmas)
    want = reference_loop(ref_dit.bfloat16(), torch.bfloat16).float()
    assert ((ours.float() - want).norm() / want.norm()).item() < 5e-2


def test_reference_fit_setup_runs_on_the_patched_trainer(ref, emu):
    """The reference's own fit-stage plumbing around the hot path, unmodified, on a trainer whose `dit` is the fused model:
    `setup_model_device_train_mode("fit")` (qwen_image_edit_trainer.py:286-330: requires_grad_ / train / LoRA filter by name),
    `configure_optimizers()` (base_trainer.py:884-916: class_path optimizer over the trainable parameters) and the DDP branch of
    `accelerator_prepare()` (:318-388: gradient checkpointing switch, AttnProcsLayers(get_lora_layers(dit)), dit.to(device));
    then one loop-body iteration must move exactly the LoRA parameters."""
    import contextlib
    import io
    import ref_common as rc
    from accelerate import Accelerator
    from qflux.losses import MseLoss
    from qflux.trainer.base_trainer import BaseTrainer
    from qflux.trainer.qwen_image_edit_trainer import QwenImageEditTrainer
    from qflux_b200 import patch_trainer
    spec = rc.CASES["qwen_hd128"]
    x = rc.rand_inputs(spec)
    dit, _ = ref.build_reference(spec)
    tr = ref._trainer(QwenImageEditTrainer, dit, MseLoss(reduction="mean"))
    tr.config = _cfg()
    tr.config.train.gradient_checkpointing = True
    tr.config.resume = None
    tr.config.validation = types.SimpleNamespace(enabled=True)
    tr.config.optimizer = types.SimpleNamespace(class_path="torch.optim.AdamW", init_args=dict(lr=1e-2, weight_decay=0.0))
    tr.config.lr_scheduler = types.SimpleNamespace(scheduler_type="constant", warmup_steps=0)
    tr.config.train.max_train_steps = 10
    tr.config.logging = types.SimpleNamespace(output_dir="/tmp")
    tr.adapter_name, tr.cache_exist, tr.use_cache = "default", True, True
    tr.vae, tr.text_encoder = torch.nn.Linear(2, 2), torch.nn.Linear(2, 2)
    tr.is_fsdp_enabled = lambda: False
    patch_trainer(tr, _host_only=True)
    with contextlib.redirect_stdout(io.StringIO()):
        QwenImageEditTrainer.setup_model_device_train_mode(tr, stage="fit")
        BaseTrainer.configure_optimizers(tr)
        BaseTrainer.accelerator_prepare(tr, train_dataloader=[1, 2, 3])
    from qflux.utils.model_summary import print_model_summary_table
    with contextlib.redirect_stdout(io.StringIO()):
        info = print_model_summary_table(tr.dit)  # fit() logs this table right before the loop (base_trainer.py:634-640)
    assert info["rows"] and info["columns"]
    names = [n for n, p in tr.dit.named_parameters() if p.requires_grad]
    assert names and all("lora" in n for n in names) and len(names) == len(list(tr.dit.parameters()))
    assert isinstance(tr.optimizer, torch.optim.AdamW) or isinstance(getattr(tr.optimizer, "optimizer", None), torch.optim.AdamW)
    before = {n: p.detach().clone() for n, p in tr.dit.named_parameters()}
    e = {k: v for k, v in x.items() if k != "u"}
    with tr.accelerator.accumulate(tr.dit):
        loss = tr._compute_loss(e)
        tr.accelerator.backward(loss)
        tr.clip_gradients()
        tr.optimizer.step()
        tr.optimizer.zero_grad()
    assert torch.isfinite(loss) and all(not torch.equal(p, before[n]) for n, p in tr.dit.named_parameters() if ".lora_A." in n)


def test_reference_train_epoch_runs_end_to_end(ref, emu, tmp_path):
    """The whole inner loop as the reference ships it: `BaseTrainer.train_epoch` (base_trainer.py:508-560) -> `training_step` ->
    `prepare_cached_embeddings` (pixel -> latent img_shapes) -> the patched `_compute_loss` -> `accelerator.backward` -> `clip_gradients`
    -> `optimizer.step` -> `lr_scheduler.step`, fed by `CachedEmbeddingLoader(reference_batch_format=True)` reading a cache that the
    reference's `EmbeddingCacheManager` wrote.  The loss must be finite every step and go down over the epoch."""
    import contextlib
    import io
    import ref_common as rc
    from qflux.data.cache_manager import EmbeddingCacheManager
    from qflux.losses import MseLoss
    from qflux.trainer.base_trainer import BaseTrainer
    from qflux.trainer.qwen_image_edit_trainer import QwenImageEditTrainer
    from qflux_b200 import patch_trainer
    from qflux_b200.cache_loader import CachedEmbeddingLoader
    spec = rc.CASES["qwen_hd128"]
    J = rc.QWEN_HD128["joint_attention_dim"]
    mgr, g = EmbeddingCacheManager(str(tmp_path)), torch.Generator().manual_seed(3)
    for i in range(4):  # the same two samples twice: a small problem the LoRA can actually fit within one epoch
        gi = torch.Generator().manual_seed(40 + i % 2)
        data = dict(image_latents=torch.randn(16, 64, generator=gi), control_latents=torch.randn(16, 64, generator=gi),
                    prompt_embeds=torch.randn(6, J, generator=gi) * 3)
        fh = dict(main_hash=f"m{i}", image_hash=f"i{i}", control_hash=f"c{i}", prompt_hash=f"p{i}")
        mgr.save_cache_embedding(data, dict(image_latents="image_hash", control_latents="control_hash", prompt_embeds="prompt_hash"), fh,
                                 img_shapes=[[3, 64, 64], [3, 64, 64]])
    dit, _ = ref.build_reference(spec)
    tr = ref._trainer(QwenImageEditTrainer, dit, MseLoss(reduction="mean"))
    tr.config, tr.adapter_name = _cfg(), "default"
    tr.config.train.max_grad_norm = 1.0
    patch_trainer(tr, _host_only=True)
    tr.optimizer = torch.optim.AdamW([p for p in tr.dit.parameters() if p.requires_grad], lr=2e-2, weight_decay=0.0)
    tr.lr_scheduler = torch.optim.lr_scheduler.ConstantLR(tr.optimizer, factor=1.0, total_iters=0)
    losses = []
    tr.training_interrupted, tr.batch_size, tr.global_step, tr.running_loss, tr.train_loss = False, 2, 0, 0.0, 0.0
    tr.fps_logger = types.SimpleNamespace(update=lambda **k: None, pause=lambda: None, resume=lambda: None, total_fps=lambda: 0.0)
    tr.update_progressbar = lambda logs: losses.append(logs["loss"])
    tr.save_checkpoint = lambda *a, **k: None
    tr.should_run_validation = lambda step: False
    torch.manual_seed(0)
    for epoch in range(6):
        loader = CachedEmbeddingLoader(str(tmp_path), batch_size=2, device="cpu", shuffle=False, reference_batch_format=True)
        with contextlib.redirect_stdout(io.StringIO()):
            BaseTrainer.train_epoch(tr, epoch, loader)
    assert len(losses) == 12 and all(l == l and abs(l) < 1e4 for l in losses), losses
    assert sum(losses[-4:]) < sum(losses[:4]), losses
