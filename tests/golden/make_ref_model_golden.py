"""Generate tests/golden/ref_model_golden_*.pt (split below 1 MB per file) by running the REFERENCE's OWN code (build container only; needs /root/reference):

    python tests/golden/make_ref_model_golden.py

What runs is /root/reference/src/qflux itself — `QwenImageTransformer2DModel`, `FluxTransformer2DModel`, the custom multi-resolution
models, `BaseTrainer.add_lora_adapter`, `QwenImageEditTrainer._compute_loss` (+ `_get_sigmas`), `FluxKontextLoraTrainer._compute_loss`
(shared and multi-resolution mode), `qflux.losses.*` — with `diffusers` / `peft` / `accelerate` replaced by the leaf restatements of
tests/shims (tests/shims/README.md).  Stored per case: the embeddings dict handed to the trainer, the noise / u / t it drew, the
model prediction, the loss and every LoRA gradient (fp32, CPU).  The GPU machine never runs this; it reads the committed .pt files.
"""
import os
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "tests", "shims"))
sys.path.insert(0, HERE)
import stub_importer  # noqa: E402

stub_importer.install()
sys.path.insert(0, "/root/reference/src")

import ref_common as rc  # noqa: E402
from accelerate import Accelerator  # noqa: E402  (tests/shims)
from diffusers.schedulers.scheduling_flow_match_euler_discrete import FlowMatchEulerDiscreteScheduler  # noqa: E402  (tests/shims)
from qflux.losses import AttentionMaskMseLoss, MaskEditLoss, MseLoss  # noqa: E402
from qflux.models.transformer_flux import FluxTransformer2DModel  # noqa: E402
from qflux.models.transformer_flux_custom import FluxTransformer2DModel as FluxCustom  # noqa: E402
from qflux.models.transformer_qwen_custom import QwenImageTransformer2DModel as QwenCustom  # noqa: E402
from qflux.models.transformer_qwenimage import QwenImageTransformer2DModel  # noqa: E402
from qflux.trainer.base_trainer import BaseTrainer  # noqa: E402
from qflux.trainer.flux_kontext_trainer import FluxKontextLoraTrainer  # noqa: E402
from qflux.trainer.qwen_image_edit_trainer import QwenImageEditTrainer  # noqa: E402
from qflux.utils.tools import pad_latents_for_multi_res  # noqa: E402


def _lora_cfg(spec):
    lora = types.SimpleNamespace(r=spec["r"], lora_alpha=spec["alpha"], init_lora_weights="gaussian", target_modules=spec["targets"],
                                 pretrained_weight=None)
    return types.SimpleNamespace(model=types.SimpleNamespace(lora=lora))


def build_reference(spec):
    cls = {"qwen": QwenImageTransformer2DModel, "flux": FluxTransformer2DModel, "flux_multi": FluxCustom, "qwen_multi": QwenCustom}[spec["kind"]]
    import contextlib
    import io
    with contextlib.redirect_stdout(io.StringIO()):  # the reference prints its config
        m = cls(**spec["cfg"])
    BaseTrainer.add_lora_adapter(m, _lora_cfg(spec), "default")   # the reference's own adapter injection (base_trainer.py:929-941)
    chk = rc.det_fill_(m, spec["seed"])
    return m, chk


def _trainer(cls, dit, criterion):
    tr = object.__new__(cls)  # no __init__: that would load encoders / pipelines
    tr.accelerator = Accelerator()
    tr.accelerator.device = torch.device("cpu")
    tr.weight_dtype = torch.float32
    tr.dit = dit
    tr.criterion = criterion
    tr.vae_scale_factor = 8
    # the Qwen-Image pipeline's scheduler: dynamic shifting => the init table is the un-shifted linspace (SURVEY.md §8c)
    tr.scheduler = FlowMatchEulerDiscreteScheduler(num_train_timesteps=1000, shift=1.0, use_dynamic_shifting=True, base_shift=0.5,
                                                   max_shift=0.9, base_image_seq_len=256, max_image_seq_len=8192)
    return tr


def run_case(name, spec):
    m, chk = build_reference(spec)
    x = rc.rand_inputs(spec)
    cap = {}
    h = m.register_forward_hook(lambda mod, a, kw, out: cap.update(pred=out[0].detach().clone(), kwargs={k: (v.detach().clone() if torch.is_tensor(v) else v) for k, v in kw.items()}),
                                with_kwargs=True)
    kind = spec["kind"]
    extra = {}
    if kind == "qwen":
        crit = MaskEditLoss(forground_weight=2.0, background_weight=1.0) if spec.get("loss") == "mask_edit" else MseLoss(reduction="mean")
        tr = _trainer(QwenImageEditTrainer, m, crit)
        # the trainer draws noise = randn_like(...) and u = compute_density_for_timestep_sampling("none") = torch.rand(B) itself
        # (qwen_image_edit_trainer.py:797-806).  The noise is reproduced by re-seeding; u is pinned to bf16-exact sigmas (ref_common.py)
        import qflux.trainer.qwen_image_edit_trainer as qt
        orig = qt.compute_density_for_timestep_sampling
        qt.compute_density_for_timestep_sampling = lambda **kw: x["u"].clone()
        try:
            torch.manual_seed(spec["seed"])
            loss = tr._compute_loss({k: v for k, v in x.items() if k != "u"})
        finally:
            qt.compute_density_for_timestep_sampling = orig
        torch.manual_seed(spec["seed"])
        extra["noise"] = torch.randn_like(x["image_latents"])
        extra["u"] = x["u"]
    elif kind == "flux":
        tr = _trainer(FluxKontextLoraTrainer, m, MseLoss(reduction="mean"))
        h_, w_ = x["hw"]
        emb = dict(x)
        emb["control_ids"] = FluxKontextLoraTrainer._prepare_latent_image_ids(1, h_, w_, torch.device("cpu"), torch.float32)
        emb["control_ids"][..., 0] = 1  # flux_kontext_trainer.py:400,419: control ids carry 1 in the first column
        emb["img_shapes"] = [[(3, h_ * 16, w_ * 16), (3, h_ * 16, w_ * 16)]] * spec["B"]
        loss = tr._compute_loss(emb)
        extra["control_ids"] = emb["control_ids"]
        extra["image_ids"] = FluxKontextLoraTrainer._prepare_latent_image_ids(1, h_, w_, torch.device("cpu"), torch.float32)
    elif kind == "flux_multi":
        tr = _trainer(FluxKontextLoraTrainer, m, AttentionMaskMseLoss(foreground_weight=2.0, background_weight=1.0, reduction="mean")
                      if spec.get("loss") == "attention_mask" else MseLoss(reduction="mean"))
        emb = {k: v for k, v in x.items() if k != "img_shapes_latent"}
        emb["timestep"] = x["timestep"].view(-1, 1)  # the multi-resolution recipe indexes [ii] and then unsqueezes dim 1 (:690-693)
        assert tr.should_use_multi_resolution_mode(emb)
        loss = tr._compute_loss(emb)
    else:  # qwen_multi: the Qwen trainer has multi-resolution disabled (qwen_image_edit_trainer.py:793); drive the custom model with the
        # FLUX trainer's recipe (flux_kontext_trainer.py:579-796): per-sample [noisy target | control], pad, mask, AttentionMaskMseLoss
        shapes = x["img_shapes_latent"]
        B, T = len(shapes), spec["T"]
        seqs, lt = [], []
        for b, sh in enumerate(shapes):
            n_t = sh[0][1] * sh[0][2]
            n_c = sum(f * hh * ww for f, hh, ww in sh[1:])
            t_ = x["timestep"][b]
            noisy = (1.0 - t_) * x["image_latents"][b, :n_t] + t_ * x["noise"][b]
            seqs.append(torch.cat([noisy, x["control_latents"][b, :n_c]], 0))
            lt.append(n_t)
        packed, img_mask = pad_latents_for_multi_res(seqs, max_seq_len=None)
        full = torch.ones(B, T + packed.shape[1], dtype=torch.bool)
        full[:, T:] = img_mask
        pred = m(hidden_states=packed, encoder_hidden_states=x["prompt_embeds"], encoder_hidden_states_mask=x["prompt_embeds_mask"],
                 timestep=x["timestep"], img_shapes=[list(s) for s in shapes], txt_seq_lens=[T] * B, attention_mask=full, return_dict=False)[0]
        Lt = max(lt)
        tmask = torch.zeros(B, Lt)
        noise_in = torch.zeros(B, Lt, 64)
        for b in range(B):
            tmask[b, : lt[b]] = 1
            noise_in[b, : lt[b]] = x["noise"][b]
        target = noise_in - x["image_latents"][:, :Lt]
        loss = AttentionMaskMseLoss(reduction="mean")(model_pred=pred[:, :Lt], target=target, attention_mask=tmask, edit_mask=None, weighting=None)
        extra.update(packed=packed, full_attention_mask=full)
    loss.backward()
    h.remove()
    # (parameters the loss does not reach — e.g. the text-stream MLP of the last block — have no .grad: stored as zeros)
    grads = {n: (p.grad.clone() if p.grad is not None else torch.zeros_like(p)) for n, p in m.named_parameters() if p.requires_grad}
    assert grads and all("lora" in n for n in grads)
    return dict(inputs=x, extra=extra, pred=cap["pred"], model_kwargs=cap["kwargs"], loss=loss.detach().clone(), grads=grads,
                weight_checksum=chk, n_params=sum(p.numel() for p in m.parameters()),
                lora_keys=sorted(grads))


def main():
    out = {}
    for name, spec in rc.CASES.items():
        out[name] = run_case(name, spec)
        c = out[name]
        print(f"{name:28s} loss={float(c['loss']):.6f} pred={tuple(c['pred'].shape)} |pred|={float(c['pred'].abs().mean()):.4f} "
              f"n_lora={len(c['grads'])} |g|={float(sum(g.norm() ** 2 for g in c['grads'].values()) ** 0.5):.4e}")
    for path in rc.save_split(out, HERE, "ref_model_golden"):
        print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
