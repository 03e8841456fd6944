"""Generate tests/golden/model_golden.pt: seeded tiny-config ORACLE outputs (pred, loss, LoRA grads) for
  * qwen_ref_tiny : the reference's own tiny test config (2 layers, heads 4x64, joint 512, rope (8,28,28);
                    /root/reference/tests/src/models/test_qwen_per_sample_rope.py:243-251)          -> pins the oracle (regression)
  * flux_ref_tiny : BASELINE config 1 (2 double + 1 single, heads 2x64 = hidden 128, joint 32, pooled 16, LoRA r=4, 64x64-px latents;
                    /root/reference/tests/src/models/test_flux_per_sample_rope.py:264-278)        -> pins the oracle (regression)
  * qwen_b200_tiny / flux_b200_tiny : head_dim-128 siblings (hidden 256) that the sm_100a kernels can run -> GPU parity fixtures
  * flux_b200_yaml_targets : the same FLUX sibling with the LoRA target regex of BASELINE config 3 (every block Linear, AdaLN linears, x_embedder)
All fp32, CPU, torch.manual_seed-free (explicit generators).  Run:  python tests/golden/make_model_golden.py
The oracle is parity-UNPINNED against diffusers (not installable offline); these vectors pin the oracle against drift and give the
GPU box an oracle-free reference.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import mmdit_oracle as mo  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ref_common as rc  # noqa: E402


def _perturb(orc, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in orc.named_parameters():
            if n.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.02)
            elif p.ndim == 1:
                p.copy_(1 + torch.randn(p.shape, generator=g) * 0.1)
        for p in orc.parameters():
            p.copy_(p.bfloat16().float())  # bf16-representable weights: the fused path stores bf16


def qwen_case(heads, hd, joint, axes, seed):
    cfg = mo.QwenConfig(num_layers=2, attention_head_dim=hd, num_attention_heads=heads, joint_attention_dim=joint, axes_dims_rope=axes)
    orc = mo.init_synthetic_(mo.QwenImageOracle(cfg), seed=seed, std=0.05)
    mo.add_lora_adapter(orc, r=4, alpha=4, b_std=0.05, seed=seed)
    _perturb(orc, seed + 1)
    g = torch.Generator().manual_seed(seed + 2)
    rn = lambda *s: torch.randn(*s, generator=g).bfloat16().float()
    B, hw, T = 2, 4, 8
    x = dict(image_latents=rn(B, hw * hw, 64), control_latents=rn(B, hw * hw, 64), prompt_embeds=rn(B, T, joint) * 3,
             prompt_embeds_mask=torch.ones(B, T, dtype=torch.int64), img_shapes=[[(1, hw, hw), (1, hw, hw)]] * B,
             noise=rn(B, hw * hw, 64), u=torch.tensor([0.5, 0.25]))
    loss, pred = mo.qwen_compute_loss(orc, **x)
    loss.backward()
    return dict(config=cfg.__dict__, state_dict={k: v.clone() for k, v in orc.state_dict().items()}, inputs=x, pred=pred.detach(),
                loss=loss.detach(), grads={n: p.grad.clone() for n, p in orc.named_parameters() if p.requires_grad})


# target_modules of BASELINE config 3 (/root/reference/configs/face_seg_flux_kontext_fp16.yaml:11): every block Linear, the AdaLN
# modulation linears and x_embedder
FLUX_YAML_TARGETS = (
    r"(.*x_embedder|.*transformer_blocks\.[0-9]+\.(norm|norm1)\.linear|.*transformer_blocks\.[0-9]+\.attn\.(to_k|to_q|to_v|to_add_out)"
    r"|.*transformer_blocks\.[0-9]+\.attn\.to_out\.0|.*single_transformer_blocks\.[0-9]+\.attn\.to_out"
    r"|.*single_transformer_blocks\.[0-9]+\.(proj_mlp|proj_out)|.*(?<!single_)transformer_blocks\.[0-9]+\.ff\.net\.2"
    r"|.*(?<!single_)transformer_blocks\.[0-9]+\.ff\.net\.0\.proj|.*(?<!single_)transformer_blocks\.[0-9]+\.norm1_context\.linear"
    r"|.*(?<!single_)transformer_blocks\.[0-9]+\.ff_context\.net\.0\.proj|.*(?<!single_)transformer_blocks\.[0-9]+\.ff_context\.net\.2"
    r"|.*(?<!single_)transformer_blocks\.[0-9]+\.attn\.(to_add_out|add_k_proj|add_q_proj|add_v_proj))")


def flux_case(heads, hd, joint, pooled, axes, seed, targets=mo.DEFAULT_TARGETS):
    cfg = mo.FluxConfig(num_layers=2, num_single_layers=1, attention_head_dim=hd, num_attention_heads=heads, joint_attention_dim=joint,
                        pooled_projection_dim=pooled, axes_dims_rope=axes, guidance_embeds=True)
    orc = mo.init_synthetic_(mo.FluxOracle(cfg), seed=seed, std=0.05)
    mo.add_lora_adapter(orc, r=4, alpha=4, target_modules=targets, b_std=0.05, seed=seed)
    _perturb(orc, seed + 1)
    g = torch.Generator().manual_seed(seed + 2)
    rn = lambda *s: torch.randn(*s, generator=g).bfloat16().float()
    B, hw, T = 1, 4, 8  # 64x64 px -> 8x8 latent -> 4x4 packed = 16 tokens per image
    x = dict(image_latents=rn(B, 16, 64), control_latents=rn(B, 16, 64), pooled=rn(B, pooled), prompt_embeds=rn(B, T, joint),
             text_ids=torch.zeros(T, 3), image_ids=mo.flux_latent_image_ids(hw, hw, 0.0), control_ids=mo.flux_latent_image_ids(hw, hw, 1.0),
             noise=rn(B, 16, 64), t=torch.tensor([0.5]))
    loss, pred = mo.flux_compute_loss_shared(orc, x["image_latents"], x["control_latents"], x["pooled"], x["prompt_embeds"], x["text_ids"],
                                             x["image_ids"], x["control_ids"], noise=x["noise"], t=x["t"])
    loss.backward()
    return dict(config=cfg.__dict__, state_dict={k: v.clone() for k, v in orc.state_dict().items()}, inputs=x, pred=pred.detach(),
                loss=loss.detach(), grads={n: p.grad.clone() for n, p in orc.named_parameters() if p.requires_grad})


def build_qwen(heads, hd, joint, axes, seed):
    """deterministic weights from seeds — the tests rebuild the model the same way instead of shipping 36 MB of state dict"""
    cfg = mo.QwenConfig(num_layers=2, attention_head_dim=hd, num_attention_heads=heads, joint_attention_dim=joint, axes_dims_rope=axes)
    orc = mo.init_synthetic_(mo.QwenImageOracle(cfg), seed=seed, std=0.05)
    mo.add_lora_adapter(orc, r=4, alpha=4, b_std=0.05, seed=seed)
    _perturb(orc, seed + 1)
    return orc


def build_flux(heads, hd, joint, pooled, axes, seed, targets=mo.DEFAULT_TARGETS):
    cfg = mo.FluxConfig(num_layers=2, num_single_layers=1, attention_head_dim=hd, num_attention_heads=heads, joint_attention_dim=joint,
                        pooled_projection_dim=pooled, axes_dims_rope=axes, guidance_embeds=True)
    orc = mo.init_synthetic_(mo.FluxOracle(cfg), seed=seed, std=0.05)
    mo.add_lora_adapter(orc, r=4, alpha=4, target_modules=targets, b_std=0.05, seed=seed)
    _perturb(orc, seed + 1)
    return orc


CASES = dict(qwen_ref_tiny=("qwen", (4, 64, 512, (8, 28, 28), 100)), flux_ref_tiny=("flux", (2, 64, 32, 16, (8, 28, 28), 200)),
             qwen_b200_tiny=("qwen", (2, 128, 128, (16, 56, 56), 300)), flux_b200_tiny=("flux", (2, 128, 64, 64, (16, 56, 56), 400)),
             flux_b200_yaml_targets=("flux", (2, 128, 64, 64, (16, 56, 56), 500, FLUX_YAML_TARGETS)))

def main():
  out = dict(qwen_ref_tiny=qwen_case(4, 64, 512, (8, 28, 28), 100), flux_ref_tiny=flux_case(2, 64, 32, 16, (8, 28, 28), 200),
             qwen_b200_tiny=qwen_case(2, 128, 128, (16, 56, 56), 300), flux_b200_tiny=flux_case(2, 128, 64, 64, (16, 56, 56), 400),
             flux_b200_yaml_targets=flux_case(2, 128, 64, 64, (16, 56, 56), 500, FLUX_YAML_TARGETS))
  # keep the fixture small: weights are rebuilt from the seeds; only a checksum is stored
  for c in out.values():
      sd = c.pop("state_dict")
      c["weight_checksum"] = float(sum(v.double().abs().sum() for v in sd.values()))
  torch.save(rc._compact(out), os.path.join(os.path.dirname(os.path.abspath(__file__)), "model_golden.pt"))  # < 1 MB
  print({k: (float(v["loss"]), v["pred"].shape) for k, v in out.items()})


if __name__ == "__main__":
    main()
