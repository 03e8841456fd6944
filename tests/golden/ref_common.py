"""Shared by tests/golden/make_ref_model_golden.py (which imports the REFERENCE's own model / trainer code) and by the tests that check
the oracle, the emulated host path and the CUDA path against the vectors it wrote.  Nothing here imports /root/reference.

Weights are a pure function of (parameter name, shape, seed): the reference model, the oracle and the fused model share the diffusers /
PEFT state-dict key names, so filling each by name gives all three identical weights without shipping them."""
import zlib

import os

import torch

DEFAULT_TARGETS = ["to_q", "to_k", "to_v", "to_out.0"]  # /root/reference/src/qflux/data/config.py:315

# every LoRA-capable Linear of the Qwen model that the fused path adapts (both streams, MLPs, AdaLN linears, embedders)
QWEN_ALL_TARGETS = (r"(img_in|txt_in|transformer_blocks\.[0-9]+\.(attn\.(to_q|to_k|to_v|add_q_proj|add_k_proj|add_v_proj|to_add_out)"
                    r"|attn\.to_out\.0|img_mlp\.net\.0\.proj|img_mlp\.net\.2|txt_mlp\.net\.0\.proj|txt_mlp\.net\.2|img_mod\.1|txt_mod\.1))")
# target_modules of BASELINE config 3 (/root/reference/configs/face_seg_flux_kontext_fp16.yaml:11)
FLUX_YAML_TARGETS = (
    r"(.*x_embedder|.*transformer_blocks\.[0-9]+\.(norm|norm1)\.linear|.*transformer_blocks\.[0-9]+\.attn\.(to_k|to_q|to_v|to_add_out)"
    r"|.*transformer_blocks\.[0-9]+\.attn\.to_out\.0|.*single_transformer_blocks\.[0-9]+\.attn\.to_out"
    r"|.*single_transformer_blocks\.[0-9]+\.(proj_mlp|proj_out)|.*(?<!single_)transformer_blocks\.[0-9]+\.ff\.net\.2"
    r"|.*(?<!single_)transformer_blocks\.[0-9]+\.ff\.net\.0\.proj|.*(?<!single_)transformer_blocks\.[0-9]+\.norm1_context\.linear"
    r"|.*(?<!single_)transformer_blocks\.[0-9]+\.ff_context\.net\.0\.proj|.*(?<!single_)transformer_blocks\.[0-9]+\.ff_context\.net\.2"
    r"|.*(?<!single_)transformer_blocks\.[0-9]+\.attn\.(to_add_out|add_k_proj|add_q_proj|add_v_proj))")

QWEN_TINY = dict(patch_size=2, in_channels=64, out_channels=16, num_layers=2, attention_head_dim=64, num_attention_heads=4,
                 joint_attention_dim=512, guidance_embeds=False, axes_dims_rope=(8, 28, 28))   # test_qwen_per_sample_rope.py:243-251
QWEN_HD128 = dict(patch_size=2, in_channels=64, out_channels=16, num_layers=2, attention_head_dim=128, num_attention_heads=2,
                  joint_attention_dim=128, guidance_embeds=False, axes_dims_rope=(16, 56, 56))
FLUX_TINY = dict(patch_size=1, in_channels=64, out_channels=64, num_layers=2, num_single_layers=1, attention_head_dim=64,
                 num_attention_heads=2, joint_attention_dim=32, pooled_projection_dim=16, guidance_embeds=False,
                 axes_dims_rope=(8, 28, 28))                                                     # test_flux_per_sample_rope.py:264-278
FLUX_HD128 = dict(patch_size=1, in_channels=64, out_channels=64, num_layers=2, num_single_layers=2, attention_head_dim=128,
                  num_attention_heads=2, joint_attention_dim=64, pooled_projection_dim=64, guidance_embeds=True,
                  axes_dims_rope=(16, 56, 56))

# name -> spec.  shapes: per-sample list of latent-patch (frame, h, w); px = pixel size per latent-patch unit (vae 8 x patch 2 = 16)
CASES = {
    # --- stock models, the trainers' own _compute_loss
    "qwen_tiny_hd64": dict(kind="qwen", cfg=QWEN_TINY, r=4, alpha=8, targets=DEFAULT_TARGETS, B=2, T=8, shapes=[(1, 4, 4), (1, 4, 4)], seed=11),
    "qwen_hd128": dict(kind="qwen", cfg=QWEN_HD128, r=4, alpha=8, targets=DEFAULT_TARGETS, B=2, T=24, shapes=[(1, 4, 4), (1, 4, 4)], seed=12),
    "qwen_hd128_plus3": dict(kind="qwen", cfg=QWEN_HD128, r=4, alpha=4, targets=DEFAULT_TARGETS, B=2, T=10,
                             shapes=[(1, 4, 4), (1, 4, 4), (1, 2, 6)], seed=13),   # Edit-Plus: target + 2 controls, frame offsets 0,1,2
    "qwen_hd128_alltargets": dict(kind="qwen", cfg=QWEN_HD128, r=4, alpha=8, targets=QWEN_ALL_TARGETS, B=2, T=24,
                                  shapes=[(1, 4, 4), (1, 4, 4)], seed=14),
    "qwen_hd128_editmask": dict(kind="qwen", cfg=QWEN_HD128, r=4, alpha=8, targets=DEFAULT_TARGETS, B=2, T=24, shapes=[(1, 4, 4), (1, 4, 4)],
                                seed=15, loss="mask_edit"),
    "flux_tiny_cfg1": dict(kind="flux", cfg=FLUX_TINY, r=4, alpha=4, targets=DEFAULT_TARGETS, B=1, T=8, hw=(4, 4), seed=21),  # BASELINE config 1
    "flux_hd128": dict(kind="flux", cfg=FLUX_HD128, r=4, alpha=8, targets=DEFAULT_TARGETS, B=2, T=8, hw=(4, 4), seed=22),
    "flux_hd128_yaml": dict(kind="flux", cfg=FLUX_HD128, r=4, alpha=8, targets=FLUX_YAML_TARGETS, B=2, T=8, hw=(4, 4), seed=23),
    # --- custom multi-resolution models (per-sample RoPE, key mask, zeroed padded rows)
    "flux_custom_multires": dict(kind="flux_multi", cfg=FLUX_HD128, r=4, alpha=8, targets=DEFAULT_TARGETS, T=8,
                                 shapes=[[(1, 4, 4), (1, 4, 4)], [(1, 2, 6), (1, 2, 6)], [(1, 6, 4), (1, 6, 4)]], seed=31,
                                 loss="attention_mask"),
    "qwen_custom_multires": dict(kind="qwen_multi", cfg=QWEN_HD128, r=4, alpha=8, targets=DEFAULT_TARGETS, T=12,
                                 shapes=[[(1, 4, 4), (1, 4, 4)], [(1, 2, 6), (1, 2, 6)], [(1, 6, 4), (1, 6, 4)]], seed=32),
}


def _gen(name: str, seed: int) -> torch.Generator:
    return torch.Generator().manual_seed((zlib.crc32(name.encode()) ^ (seed * 2654435761)) & 0x7FFFFFFF)


def bf16_exact(t: torch.Tensor) -> torch.Tensor:
    return t.bfloat16().float()


@torch.no_grad()
def det_fill_(model: torch.nn.Module, seed: int, w_std: float = 0.05, lora_b_std: float = 0.05) -> float:
    """Fill every parameter from its NAME (bf16-representable values; the fused path stores bf16).  Returns a checksum."""
    tot = 0.0
    for name, p in sorted(model.named_parameters(), key=lambda kv: kv[0]):
        name = name.replace(".base_layer.", ".")  # PEFT wraps adapted Linears: the frozen weight keeps its diffusers name here
        g = _gen(name, seed)
        r = torch.randn(p.shape, generator=g, dtype=torch.float32)
        if ".lora_A." in name:
            v = r / p.shape[0]                 # PEFT "gaussian": std 1/r
        elif ".lora_B." in name:
            v = r * lora_b_std                 # non-zero so that dA != 0
        elif name.endswith("bias"):
            v = r * 0.02
        elif p.ndim == 1:
            v = 1.0 + 0.1 * r                  # norm weights
        else:
            v = r * w_std
        v = bf16_exact(v)
        p.copy_(v.to(p.dtype))
        tot += float(v.double().abs().sum())
    return tot


def rand_inputs(spec: dict) -> dict:
    """Deterministic, bf16-representable inputs of one case (reference `embeddings` keys)."""
    g = torch.Generator().manual_seed(1000 + spec["seed"])
    rn = lambda *s: bf16_exact(torch.randn(*s, generator=g))
    kind, cfg, T = spec["kind"], spec["cfg"], spec["T"]
    J = cfg["joint_attention_dim"]
    if kind == "qwen":
        B, shapes = spec["B"], spec["shapes"]
        L = shapes[0][1] * shapes[0][2]
        Lc = sum(f * h * w for f, h, w in shapes[1:])
        # u -> idx = (u * 1000).long() -> sigma = (1000 - idx) / 1000 in {0.5, 0.25, 0.75, 0.125}: bf16-exact, because the model rounds
        # sigma to the working dtype before the 1000x sinusoid (transformer_qwenimage.py:624) and the fused path works in bf16
        x = dict(image_latents=rn(B, L, 64), control_latents=rn(B, Lc, 64), prompt_embeds=rn(B, T, J) * 3,
                 prompt_embeds_mask=torch.ones(B, T, dtype=torch.int64), img_shapes=[list(shapes)] * B,
                 u=torch.tensor([0.5, 0.75, 0.25, 0.875][:B]))
        if spec.get("loss") == "mask_edit":
            x["edit_mask"] = (torch.rand(B, L, generator=g) > 0.5).float()
        return x
    if kind == "flux":
        B, (h, w) = spec["B"], spec["hw"]
        L = h * w
        return dict(image_latents=rn(B, L, 64), control_latents=rn(B, L, 64), pooled_prompt_embeds=rn(B, cfg["pooled_projection_dim"]),
                    prompt_embeds=rn(B, T, J), text_ids=torch.zeros(T, 3), image=torch.zeros(B, 3, h * 16, w * 16),
                    # t with t * 1000 exact in bf16: a bf16 FLUX model multiplies the timestep by 1000 in bf16 (transformer_flux.py:707-710)
                    noise=rn(B, L, 64), timestep=torch.tensor([0.5, 0.25, 0.125][:B]), hw=(h, w))
    shapes = spec["shapes"]
    B = len(shapes)
    lt = [s[0][1] * s[0][2] for s in shapes]
    lc = [sum(f * h * w for f, h, w in s[1:]) for s in shapes]
    Lt, Lc = max(lt), max(lc)
    x0, ctrl = torch.zeros(B, Lt, 64), torch.zeros(B, Lc, 64)
    noise = []
    for b in range(B):
        x0[b, : lt[b]] = rn(lt[b], 64)
        ctrl[b, : lc[b]] = rn(lc[b], 64)
        noise.append(rn(lt[b], 64))
    x = dict(image_latents=x0, control_latents=ctrl, prompt_embeds=rn(B, T, J) * (1 if kind == "flux_multi" else 3),
             noise=noise, timestep=torch.tensor([0.5, 0.25, 0.125][:B]), img_shapes_latent=[list(s) for s in shapes],
             # pixel-space shapes as the dataset delivers them: (3, H, W) with H = 16 h
             img_shapes=[[(3, h * 16, w * 16) for (_, h, w) in s] for s in shapes])
    if kind == "flux_multi":
        x.update(pooled_prompt_embeds=rn(B, cfg["pooled_projection_dim"]), text_ids=torch.zeros(T, 3))
    else:
        x["prompt_embeds_mask"] = torch.ones(B, T, dtype=torch.int64)
    return x


def rel_l2(a: torch.Tensor, b: torch.Tensor) -> float:
    a, b = a.double(), b.double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


# ------------------------------------------------------------------------------------------------ golden files
GOLDEN_PART_BYTES = 900_000  # every stored file stays below 1 MB


def _compact(o):
    """Deep copy with every tensor cloned: a saved view would drag its whole base storage into the file."""
    if torch.is_tensor(o):
        return o.clone()
    if isinstance(o, dict):
        return {k: _compact(v) for k, v in o.items()}
    if isinstance(o, (list, tuple)):
        return type(o)(_compact(v) for v in o)
    return o


def save_split(cases: dict, directory: str, stem: str) -> list:
    """torch.save the per-case dict as stem_0.pt, stem_1.pt, ... (whole cases per file, each file < GOLDEN_PART_BYTES)."""
    import io
    parts, cur, cur_bytes = [], {}, 0
    for name, c in cases.items():
        c = _compact(c)
        buf = io.BytesIO()
        torch.save(c, buf)
        n = len(buf.getvalue())
        assert n < GOLDEN_PART_BYTES, f"golden case {name} alone is {n} bytes"
        if cur and cur_bytes + n > GOLDEN_PART_BYTES:
            parts.append(cur)
            cur, cur_bytes = {}, 0
        cur[name], cur_bytes = c, cur_bytes + n
    if cur:
        parts.append(cur)
    for f in os.listdir(directory):
        if f.startswith(stem + "_") and f.endswith(".pt"):
            os.remove(os.path.join(directory, f))
    paths = []
    for i, part in enumerate(parts):
        paths.append(os.path.join(directory, f"{stem}_{i}.pt"))
        torch.save(part, paths[-1])
    return paths


def load_split(directory: str, stem: str) -> dict:
    out = {}
    names = sorted(f for f in os.listdir(directory) if f.startswith(stem + "_") and f.endswith(".pt"))
    assert names, f"no {stem}_*.pt in {directory}"
    for f in names:
        out.update(torch.load(os.path.join(directory, f), weights_only=False))
    return out
