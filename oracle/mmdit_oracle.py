"""ORACLE — test infrastructure only.  PARITY PINNED to the reference's own code through leaf restatements of diffusers / peft.

CPU/GPU-agnostic pure-torch restatement of the reference's hot path (SURVEY.md §8a):

    noise-predict forward (Qwen-Image / FLUX MMDiT) -> flow-matching MSE -> backward (LoRA grads)

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference` / library-baseline legs may
import this file.  The product path (qflux_b200) never routes through it.

How it is pinned: the arithmetic of this path lives partly in `diffusers` / `peft`, which are not vendored in /root/reference and
are not installable here (no network).  tests/shims/ restates ONLY the leaf layers those packages contribute (RMSNorm, AdaLayerNorm*,
FeedForward, Timesteps/TimestepEmbedding, Attention container, SDPA dispatch, rotary helpers, PEFT LoRA Linear, scheduler tables);
with them, tests/golden/make_ref_model_golden.py runs the REFERENCE'S OWN `qflux.models.transformer_qwenimage`, `transformer_flux`,
`transformer_qwen_custom`, `transformer_flux_custom`, `BaseTrainer.add_lora_adapter`, `QwenImageEditTrainer._compute_loss` and
`FluxKontextLoraTrainer._compute_loss` (shared + multi-resolution) and commits their outputs (tests/golden/ref_model_golden_*.pt).
tests/test_reference_goldens.py holds this file to those vectors at fp32 round-off (pred / loss 1e-5, every LoRA gradient 1e-4) on
ten cases (stock + custom models, Edit-Plus 3-image RoPE, every LoRA target set, all three losses).  What remains un-pinned is the
dozen leaf ops of tests/shims (no diffusers wheel exists offline to check them against); the loss functions are pinned directly to
`qflux.losses` (tests/test_oracle_losses.py).

Reference files followed (paths relative to /root/reference/src/qflux):
  models/transformer_qwenimage.py:93-140   apply_rotary_emb_qwen (complex, pairs (2i,2i+1))
  models/transformer_qwenimage.py:143-156  QwenTimestepProjEmbeddings (Timesteps scale=1000)
  models/transformer_qwenimage.py:159-254  QwenEmbedRope (scale_rope=True, per-image frame offset)
  models/transformer_qwenimage.py:257-354  QwenDoubleStreamAttnProcessor2_0 (joint [txt; img] attention)
  models/transformer_qwenimage.py:377-494  QwenImageTransformerBlock (AdaLN-Zero x2 streams, GELU-tanh MLP)
  models/transformer_qwenimage.py:497-672  QwenImageTransformer2DModel.forward
  models/transformer_qwen_custom.py:86-216,384-573   per-sample RoPE, padded-row zeroing and additive key mask of the custom Qwen forward
  models/transformer_flux_custom.py:84-160,372-741   the same for FLUX (per-sample ids, identity rotation on padding)
  models/transformer_flux.py:102-166       FluxAttnProcessor (RoPE applied after concat)
  models/transformer_flux.py:385-523       FluxSingleTransformerBlock / FluxTransformerBlock
  models/transformer_flux.py:526-554       FluxPosEmbed
  models/transformer_flux.py:611-828       FluxTransformer2DModel
  trainer/qwen_image_edit_trainer.py:777-861   _compute_loss / _get_sigmas
  trainer/flux_kontext_trainer.py:494-577      _compute_loss_shared_mode
  trainer/base_trainer.py:929-941              add_lora_adapter (peft LoraConfig: r, alpha, "gaussian")
State-dict key names equal diffusers' (and PEFT's `base_layer` / `lora_A.default` / `lora_B.default`) so real
checkpoints load unchanged when they become available.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch
import torch.nn as nn
import torch.nn.functional as F


# ----------------------------------------------------------------------------------------------------------------
# small building blocks (diffusers / peft semantics, SURVEY.md §8c)
# ----------------------------------------------------------------------------------------------------------------
class LoraLinear(nn.Module):
    """`nn.Linear` that can carry one PEFT-style LoRA adapter.

    Without an adapter the parameter names are `weight` / `bias` (diffusers).  After `add_adapter` they are
    `base_layer.weight`, `base_layer.bias`, `lora_A.default.weight` [r,in], `lora_B.default.weight` [out,r]
    (PEFT `LoraLayer`), and  y = base(x) + lora_B(lora_A(x)) * (alpha / r)   (dropout 0).
    """

    def __init__(self, in_features: int, out_features: int, bias: bool = True):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.base_layer = nn.Linear(in_features, out_features, bias=bias)
        self.lora_A = nn.ModuleDict()
        self.lora_B = nn.ModuleDict()
        self.scaling = 0.0
        self.r = 0
        self._register_state_dict_hook(LoraLinear._sd_hook)

    # expose diffusers names (`weight`, `bias`) when no adapter is attached
    @staticmethod
    def _sd_hook(module, state_dict, prefix, local_metadata):
        if module.r == 0:
            for n in ("weight", "bias"):
                k = prefix + "base_layer." + n
                if k in state_dict:
                    state_dict[prefix + n] = state_dict.pop(k)

    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        for n in ("weight", "bias"):
            if prefix + n in state_dict:
                state_dict[prefix + "base_layer." + n] = state_dict.pop(prefix + n)
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)

    def add_adapter(self, r: int, alpha: float, init: str = "gaussian", generator: torch.Generator | None = None,
                    b_std: float = 0.0):
        w = self.base_layer.weight
        a = nn.Linear(self.in_features, r, bias=False).to(device=w.device, dtype=w.dtype)
        b = nn.Linear(r, self.out_features, bias=False).to(device=w.device, dtype=w.dtype)
        with torch.no_grad():
            if init == "gaussian":  # peft: nn.init.normal_(A, std=1/r); B zeros
                a.weight.copy_(torch.randn(a.weight.shape, generator=generator, dtype=torch.float32) / r)
            else:  # peft default: kaiming_uniform(a=sqrt(5))
                bound = 1.0 / math.sqrt(self.in_features)
                a.weight.copy_((torch.rand(a.weight.shape, generator=generator, dtype=torch.float32) * 2 - 1) * bound)
            if b_std > 0:  # synthetic benches use a non-zero B so that dA != 0 (SURVEY.md §8d cfg 2)
                b.weight.copy_(torch.randn(b.weight.shape, generator=generator, dtype=torch.float32) * b_std)
            else:
                b.weight.zero_()
        self.lora_A["default"], self.lora_B["default"] = a, b
        self.r, self.scaling = r, alpha / r
        self.base_layer.requires_grad_(False)

    def forward(self, x):
        y = self.base_layer(x)
        if self.r:
            y = y + self.lora_B["default"](self.lora_A["default"](x)) * self.scaling
        return y


def diffusers_rms_norm(x: torch.Tensor, weight: torch.Tensor | None, eps: float) -> torch.Tensor:
    """diffusers `RMSNorm.forward`: variance in fp32, cast to the weight dtype BEFORE the weight multiply."""
    in_dtype = x.dtype
    var = x.to(torch.float32).pow(2).mean(-1, keepdim=True)
    x = x * torch.rsqrt(var + eps)  # fp32 result (promotion)
    if weight is not None:
        if weight.dtype in (torch.float16, torch.bfloat16):
            x = x.to(weight.dtype)
        x = x * weight
    else:
        x = x.to(in_dtype)
    return x


class DiffusersRMSNorm(nn.Module):
    def __init__(self, dim, eps=1e-6):
        super().__init__()
        self.eps = eps
        self.weight = nn.Parameter(torch.ones(dim))

    def forward(self, x):
        return diffusers_rms_norm(x, self.weight, self.eps)


def timestep_sinusoid(t: torch.Tensor, dim: int = 256, scale: float = 1.0, max_period: int = 10000) -> torch.Tensor:
    """diffusers `Timesteps(dim, flip_sin_to_cos=True, downscale_freq_shift=0, scale)` — fp32 freqs, [cos, sin]."""
    half = dim // 2
    exponent = -math.log(max_period) * torch.arange(half, dtype=torch.float32, device=t.device) / half
    emb = t[:, None].float() * torch.exp(exponent)[None, :]
    emb = scale * emb
    return torch.cat([torch.cos(emb), torch.sin(emb)], dim=-1)


class TimestepEmbedding(nn.Module):
    def __init__(self, in_ch, dim):
        super().__init__()
        self.linear_1 = nn.Linear(in_ch, dim)
        self.linear_2 = nn.Linear(dim, dim)

    def forward(self, x):
        return self.linear_2(F.silu(self.linear_1(x)))


class FeedForward(nn.Module):
    """diffusers FeedForward(dim, dim_out=dim, activation_fn="gelu-approximate"): net.0.proj, net.2."""

    def __init__(self, dim, mult=4):
        super().__init__()
        proj = nn.Module()
        proj.proj = LoraLinear(dim, dim * mult)
        self.net = nn.ModuleList([proj, nn.Identity(), LoraLinear(dim * mult, dim)])

    def forward(self, x):
        return self.net[2](F.gelu(self.net[0].proj(x), approximate="tanh"))


class JointAttention(nn.Module):
    """diffusers Attention(query_dim=D, added_kv_proj_dim=D, qk_norm='rms_norm', bias=True) parameter container."""

    def __init__(self, dim, heads, head_dim, eps=1e-6, added=True, pre_only=False, torch_rms=False):
        super().__init__()
        self.heads, self.head_dim = heads, head_dim
        self.to_q, self.to_k, self.to_v = LoraLinear(dim, dim), LoraLinear(dim, dim), LoraLinear(dim, dim)
        norm = (lambda: nn.RMSNorm(head_dim, eps=eps)) if torch_rms else (lambda: DiffusersRMSNorm(head_dim, eps))
        self.norm_q, self.norm_k = norm(), norm()
        if not pre_only:
            self.to_out = nn.ModuleList([LoraLinear(dim, dim), nn.Identity()])
        if added:
            self.add_q_proj, self.add_k_proj, self.add_v_proj = LoraLinear(dim, dim), LoraLinear(dim, dim), LoraLinear(dim, dim)
            self.norm_added_q, self.norm_added_k = norm(), norm()
            self.to_add_out = LoraLinear(dim, dim)


def sdpa(q, k, v, attn_mask=None):
    """dispatch_attention_fn(backend=None): F.scaled_dot_product_attention on [B,H,S,d], scale 1/sqrt(d)."""
    o = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), attn_mask=attn_mask)
    return o.transpose(1, 2)


# ----------------------------------------------------------------------------------------------------------------
# Qwen-Image
# ----------------------------------------------------------------------------------------------------------------
def apply_rotary_emb_qwen(x: torch.Tensor, freqs_cis: torch.Tensor) -> torch.Tensor:
    """transformer_qwenimage.py:134-140 (use_real=False): complex multiply in fp32, cast back."""
    xc = torch.view_as_complex(x.float().reshape(*x.shape[:-1], -1, 2))
    out = torch.view_as_real(xc * freqs_cis.unsqueeze(1)).flatten(3)
    return out.type_as(x)


class QwenEmbedRope:
    """transformer_qwenimage.py:159-254 with scale_rope=True."""

    def __init__(self, theta: int, axes_dim: list[int]):
        self.theta, self.axes_dim = theta, axes_dim
        pos = torch.arange(4096)
        neg = torch.arange(4096).flip(0) * -1 - 1
        self.pos_freqs = torch.cat([self._params(pos, d) for d in axes_dim], dim=1)
        self.neg_freqs = torch.cat([self._params(neg, d) for d in axes_dim], dim=1)

    def _params(self, index, dim):
        freqs = torch.outer(index, 1.0 / torch.pow(self.theta, torch.arange(0, dim, 2).to(torch.float32).div(dim)))
        return torch.polar(torch.ones_like(freqs), freqs)

    def video_freqs(self, frame, height, width, idx):
        fp = self.pos_freqs.split([x // 2 for x in self.axes_dim], dim=1)
        fn = self.neg_freqs.split([x // 2 for x in self.axes_dim], dim=1)
        f_f = fp[0][idx: idx + frame].view(frame, 1, 1, -1).expand(frame, height, width, -1)
        f_h = torch.cat([fn[1][-(height - height // 2):], fp[1][: height // 2]], dim=0)
        f_h = f_h.view(1, height, 1, -1).expand(frame, height, width, -1)
        f_w = torch.cat([fn[2][-(width - width // 2):], fp[2][: width // 2]], dim=0)
        f_w = f_w.view(1, 1, width, -1).expand(frame, height, width, -1)
        return torch.cat([f_f, f_h, f_w], dim=-1).reshape(frame * height * width, -1).clone().contiguous()

    def __call__(self, video_fhw, txt_seq_lens, device):
        if isinstance(video_fhw, list):
            video_fhw = video_fhw[0]  # shared mode: only img_shapes[0] is used (:206-207)
        if not isinstance(video_fhw, list):
            video_fhw = [video_fhw]
        vid, max_vid_index = [], 0
        for idx, (frame, height, width) in enumerate(video_fhw):
            vid.append(self.video_freqs(frame, height, width, idx))
            max_vid_index = max(height // 2, width // 2, max_vid_index)
        max_len = max(txt_seq_lens)
        txt = self.pos_freqs[max_vid_index: max_vid_index + max_len]
        return torch.cat(vid, dim=0).to(device), txt.to(device)


def qwen_rope_per_sample(q, k, rope_list, T, img_offset="aligned"):
    """QwenDoubleStreamAttnProcessorPerSample._apply_rope_per_sample (transformer_qwen_custom.py:167-216) on the joint [text; image]
    sequence: sample b rotates its first txt_len_b positions with its text table and L_b positions with its image table; all other
    positions (padding) keep the identity rotation.
    img_offset: where the image table is applied.  "reference" = joint positions [txt_len_b, txt_len_b + L_b) — what the reference does
    (:199-208: `seq_txt` is the per-sample text length, not the padded one), which is mis-aligned by T - txt_len_b whenever a sample's
    text is padded; "aligned" = [T, T + L_b), the positions the image tokens actually occupy.  The two agree when no text is padded
    (the only case the reference's tests cover, tests/src/models/test_qwen_per_sample_rope.py); the fused path implements "aligned",
    which is what makes a padded batch equal the per-sample un-padded runs."""
    qo, ko = q.clone(), k.clone()
    for b, (img_f, txt_f) in enumerate(rope_list):
        nt, ni = txt_f.shape[0], img_f.shape[0]
        i0 = T if img_offset == "aligned" else nt
        for src, dst in ((q, qo), (k, ko)):
            dst[b:b + 1, :nt] = apply_rotary_emb_qwen(src[b:b + 1, :nt], txt_f)
            dst[b:b + 1, i0:i0 + ni] = apply_rotary_emb_qwen(src[b:b + 1, i0:i0 + ni], img_f)
    return qo, ko


class QwenBlock(nn.Module):
    def __init__(self, dim, heads, head_dim, eps=1e-6):
        super().__init__()
        self.eps, self.dim = eps, dim
        self.img_mod = nn.Sequential(nn.SiLU(), LoraLinear(dim, 6 * dim))
        self.txt_mod = nn.Sequential(nn.SiLU(), LoraLinear(dim, 6 * dim))
        self.attn = JointAttention(dim, heads, head_dim, eps)
        self.img_mlp, self.txt_mlp = FeedForward(dim), FeedForward(dim)

    def _ln(self, x):
        return F.layer_norm(x, (self.dim,), None, None, self.eps)

    @staticmethod
    def _modulate(x, mod):
        shift, scale, gate = mod.chunk(3, dim=-1)
        return x * (1 + scale.unsqueeze(1)) + shift.unsqueeze(1), gate.unsqueeze(1)

    def forward(self, hidden, enc, temb, rope, attn_mask=None, img_offset="aligned"):
        """rope: (img_freqs, txt_freqs) shared by the batch, or a LIST of such pairs, one per sample (custom model,
        transformer_qwen_custom.py:167-216).  attn_mask: additive [B,1,1,S] key mask (:507-517)."""
        a = self.attn
        img_mod1, img_mod2 = self.img_mod(temb).chunk(2, dim=-1)
        txt_mod1, txt_mod2 = self.txt_mod(temb).chunk(2, dim=-1)
        img_m, img_g1 = self._modulate(self._ln(hidden), img_mod1)
        txt_m, txt_g1 = self._modulate(self._ln(enc), txt_mod1)
        T = enc.shape[1]
        H = a.heads
        iq, ik, iv = (f(img_m).unflatten(-1, (H, -1)) for f in (a.to_q, a.to_k, a.to_v))
        tq, tk, tv = (f(txt_m).unflatten(-1, (H, -1)) for f in (a.add_q_proj, a.add_k_proj, a.add_v_proj))
        iq, ik, tq, tk = a.norm_q(iq), a.norm_k(ik), a.norm_added_q(tq), a.norm_added_k(tk)
        if isinstance(rope, list):
            q, k, v = torch.cat([tq, iq], 1), torch.cat([tk, ik], 1), torch.cat([tv, iv], 1)
            q, k = qwen_rope_per_sample(q, k, rope, T, img_offset)
        else:
            img_f, txt_f = rope
            iq, ik = apply_rotary_emb_qwen(iq, img_f), apply_rotary_emb_qwen(ik, img_f)
            tq, tk = apply_rotary_emb_qwen(tq, txt_f), apply_rotary_emb_qwen(tk, txt_f)
            q, k, v = torch.cat([tq, iq], 1), torch.cat([tk, ik], 1), torch.cat([tv, iv], 1)
        o = sdpa(q, k, v, attn_mask).flatten(2, 3).to(q.dtype)  # NB: encoder_hidden_states_mask is never used (:276)
        txt_o, img_o = a.to_add_out(o[:, :T]), a.to_out[0](o[:, T:])
        hidden = hidden + img_g1 * img_o
        enc = enc + txt_g1 * txt_o
        img_m2, img_g2 = self._modulate(self._ln(hidden), img_mod2)
        hidden = hidden + img_g2 * self.img_mlp(img_m2)
        txt_m2, txt_g2 = self._modulate(self._ln(enc), txt_mod2)
        enc = enc + txt_g2 * self.txt_mlp(txt_m2)
        return enc, hidden


class AdaLayerNormContinuous(nn.Module):
    """diffusers AdaLayerNormContinuous(D, D, elementwise_affine=False, eps=1e-6): chunk order (scale, shift)."""

    def __init__(self, dim, eps=1e-6):
        super().__init__()
        self.dim, self.eps = dim, eps
        self.linear = LoraLinear(dim, 2 * dim)

    def forward(self, x, temb):
        emb = self.linear(F.silu(temb).to(x.dtype))
        scale, shift = emb.chunk(2, dim=1)
        return F.layer_norm(x, (self.dim,), None, None, self.eps) * (1 + scale)[:, None, :] + shift[:, None, :]


@dataclass
class QwenConfig:
    patch_size: int = 2
    in_channels: int = 64
    out_channels: int = 16
    num_layers: int = 60
    attention_head_dim: int = 128
    num_attention_heads: int = 24
    joint_attention_dim: int = 3584
    guidance_embeds: bool = False
    axes_dims_rope: tuple = (16, 56, 56)


class QwenImageOracle(nn.Module):
    def __init__(self, cfg: QwenConfig):
        super().__init__()
        self.config = cfg
        D = cfg.num_attention_heads * cfg.attention_head_dim
        self.inner_dim = D
        self.pos_embed = QwenEmbedRope(10000, list(cfg.axes_dims_rope))
        tte = nn.Module()
        tte.timestep_embedder = TimestepEmbedding(256, D)
        self.time_text_embed = tte
        self.txt_norm = DiffusersRMSNorm(cfg.joint_attention_dim, 1e-6)
        self.img_in = LoraLinear(cfg.in_channels, D)
        self.txt_in = LoraLinear(cfg.joint_attention_dim, D)
        self.transformer_blocks = nn.ModuleList(
            [QwenBlock(D, cfg.num_attention_heads, cfg.attention_head_dim) for _ in range(cfg.num_layers)])
        self.norm_out = AdaLayerNormContinuous(D)
        self.proj_out = LoraLinear(D, cfg.patch_size ** 2 * cfg.out_channels)

    def forward(self, hidden_states, encoder_hidden_states=None, encoder_hidden_states_mask=None, timestep=None,
                img_shapes=None, txt_seq_lens=None, guidance=None, attention_kwargs=None, return_dict=False, attention_mask=None,
                img_offset="aligned"):
        """The stock forward (transformer_qwenimage.py:570-672) and, with `attention_mask` [B, T + L] / per-sample `img_shapes`
        (a list of lists whose entries differ), the custom multi-resolution forward (transformer_qwen_custom.py:384-573): per-sample
        RoPE, padded rows zeroed after the embedders and after every block, additive -inf key mask, padded output rows zeroed."""
        h = self.img_in(hidden_states)
        timestep = timestep.to(h.dtype)  # bf16 rounding of sigma happens HERE (:624)
        enc = self.txt_in(self.txt_norm(encoder_hidden_states))
        temb = self.time_text_embed.timestep_embedder(timestep_sinusoid(timestep, 256, scale=1000.0).to(h.dtype))
        nested = isinstance(img_shapes, list) and len(img_shapes) > 0 and isinstance(img_shapes[0], list)
        if nested and not all(sh == img_shapes[0] for sh in img_shapes):  # :458-474 per-sample mode only when the samples differ
            lens = txt_seq_lens if isinstance(txt_seq_lens, list) else [txt_seq_lens] * len(img_shapes)
            rope = [self.pos_embed([sh], [n], h.device) for sh, n in zip(img_shapes, lens)]
        else:
            rope = self.pos_embed(img_shapes, txt_seq_lens, h.device)
        add_mask = img_valid = None
        if attention_mask is not None:
            m = attention_mask.to(h.device) > 0
            T = enc.shape[1]
            img_valid = m[:, T:T + h.shape[1]]
            enc = enc.masked_fill(~m[:, :T].unsqueeze(-1), 0)
            h = h.masked_fill(~img_valid.unsqueeze(-1), 0)
            add_mask = torch.zeros(m.shape[0], 1, 1, m.shape[1], dtype=h.dtype, device=h.device).masked_fill(~m[:, None, None, :], float("-inf"))
        for blk in self.transformer_blocks:
            enc, h = blk(h, enc, temb, rope, add_mask, img_offset)
            if img_valid is not None:
                h = h * img_valid.unsqueeze(-1)  # :545-560
        out = self.proj_out(self.norm_out(h, temb))
        if img_valid is not None:
            out = out.masked_fill(~img_valid.unsqueeze(-1), 0)
        return (out,)


# ----------------------------------------------------------------------------------------------------------------
# FLUX.1 (Kontext)
# ----------------------------------------------------------------------------------------------------------------
def flux_rope(ids: torch.Tensor, axes_dim, theta=10000):
    """FluxPosEmbed.forward (transformer_flux.py:533-554): float64 freqs -> fp32 cos/sin, repeat_interleave(2)."""
    cos_o, sin_o = [], []
    pos = ids.float()
    for i, d in enumerate(axes_dim):
        freqs = 1.0 / (theta ** (torch.arange(0, d, 2, dtype=torch.float64, device=ids.device)[: d // 2] / d))
        fr = torch.outer(pos[:, i], freqs)
        cos_o.append(fr.cos().repeat_interleave(2, dim=1).float())
        sin_o.append(fr.sin().repeat_interleave(2, dim=1).float())
    return torch.cat(cos_o, -1), torch.cat(sin_o, -1)


def apply_rotary_emb_real(x, cos, sin):
    """diffusers apply_rotary_emb(use_real=True, unbind_dim=-1, sequence_dim=1); x [B,S,H,d], cos/sin [S,d]."""
    cos, sin = (cos[None, :, None, :], sin[None, :, None, :]) if cos.ndim == 2 else (cos[:, :, None, :], sin[:, :, None, :])  # [B,S,d]: per sample
    xr, xi = x.reshape(*x.shape[:-1], -1, 2).unbind(-1)
    xrot = torch.stack([-xi, xr], dim=-1).flatten(3)
    return (x.float() * cos + xrot.float() * sin).to(x.dtype)


class AdaLayerNormZero(nn.Module):
    def __init__(self, dim, n_chunks=6):
        super().__init__()
        self.dim, self.n = dim, n_chunks
        self.linear = LoraLinear(dim, n_chunks * dim)

    def forward(self, x, emb):
        parts = self.linear(F.silu(emb)).chunk(self.n, dim=1)
        shift, scale = parts[0], parts[1]
        x = F.layer_norm(x, (self.dim,), None, None, 1e-6) * (1 + scale[:, None]) + shift[:, None]
        return (x,) + tuple(parts[2:])


class FluxDoubleBlock(nn.Module):
    def __init__(self, dim, heads, head_dim):
        super().__init__()
        self.dim = dim
        self.norm1, self.norm1_context = AdaLayerNormZero(dim), AdaLayerNormZero(dim)
        self.attn = JointAttention(dim, heads, head_dim, torch_rms=True)
        self.ff, self.ff_context = FeedForward(dim), FeedForward(dim)

    def forward(self, hidden, enc, temb, rope, attn_mask=None):
        a, H = self.attn, self.attn.heads
        nh, gate_msa, shift_mlp, scale_mlp, gate_mlp = self.norm1(hidden, temb)
        ne, c_gate_msa, c_shift_mlp, c_scale_mlp, c_gate_mlp = self.norm1_context(enc, temb)
        q, k, v = (f(nh).unflatten(-1, (H, -1)) for f in (a.to_q, a.to_k, a.to_v))
        q, k = a.norm_q(q), a.norm_k(k)
        eq, ek, ev = (f(ne).unflatten(-1, (H, -1)) for f in (a.add_q_proj, a.add_k_proj, a.add_v_proj))
        eq, ek = a.norm_added_q(eq), a.norm_added_k(ek)
        q, k, v = torch.cat([eq, q], 1), torch.cat([ek, k], 1), torch.cat([ev, v], 1)
        q, k = apply_rotary_emb_real(q, *rope), apply_rotary_emb_real(k, *rope)
        o = sdpa(q, k, v, attn_mask).flatten(2, 3).to(q.dtype)
        T = enc.shape[1]
        ctx_o, img_o = a.to_add_out(o[:, :T]), a.to_out[0](o[:, T:])
        hidden = hidden + gate_msa.unsqueeze(1) * img_o
        n2 = F.layer_norm(hidden, (self.dim,), None, None, 1e-6) * (1 + scale_mlp[:, None]) + shift_mlp[:, None]
        hidden = hidden + gate_mlp.unsqueeze(1) * self.ff(n2)
        enc = enc + c_gate_msa.unsqueeze(1) * ctx_o
        n2c = F.layer_norm(enc, (self.dim,), None, None, 1e-6) * (1 + c_scale_mlp[:, None]) + c_shift_mlp[:, None]
        enc = enc + c_gate_mlp.unsqueeze(1) * self.ff_context(n2c)
        return enc, hidden


class FluxSingleBlock(nn.Module):
    def __init__(self, dim, heads, head_dim, mlp_ratio=4.0):
        super().__init__()
        self.norm = AdaLayerNormZero(dim, n_chunks=3)
        self.proj_mlp = LoraLinear(dim, int(dim * mlp_ratio))
        self.proj_out = LoraLinear(dim + int(dim * mlp_ratio), dim)
        self.attn = JointAttention(dim, heads, head_dim, added=False, pre_only=True, torch_rms=True)

    def forward(self, hidden, enc, temb, rope, attn_mask=None):
        T = enc.shape[1]
        x = torch.cat([enc, hidden], dim=1)
        n, gate = self.norm(x, temb)
        mlp = F.gelu(self.proj_mlp(n), approximate="tanh")
        a, H = self.attn, self.attn.heads
        q, k, v = (f(n).unflatten(-1, (H, -1)) for f in (a.to_q, a.to_k, a.to_v))
        q, k = apply_rotary_emb_real(a.norm_q(q), *rope), apply_rotary_emb_real(a.norm_k(k), *rope)
        o = sdpa(q, k, v, attn_mask).flatten(2, 3).to(q.dtype)
        x = x + gate.unsqueeze(1) * self.proj_out(torch.cat([o, mlp], dim=2))
        return x[:, :T], x[:, T:]


@dataclass
class FluxConfig:
    patch_size: int = 1
    in_channels: int = 64
    out_channels: int | None = None
    num_layers: int = 19
    num_single_layers: int = 38
    attention_head_dim: int = 128
    num_attention_heads: int = 24
    joint_attention_dim: int = 4096
    pooled_projection_dim: int = 768
    guidance_embeds: bool = False
    axes_dims_rope: tuple = (16, 56, 56)


class FluxOracle(nn.Module):
    def __init__(self, cfg: FluxConfig):
        super().__init__()
        self.config = cfg
        D = cfg.num_attention_heads * cfg.attention_head_dim
        self.inner_dim = D
        tte = nn.Module()
        tte.timestep_embedder = TimestepEmbedding(256, D)
        if cfg.guidance_embeds:
            tte.guidance_embedder = TimestepEmbedding(256, D)
        tte.text_embedder = TimestepEmbedding(cfg.pooled_projection_dim, D)  # PixArtAlphaTextProjection(act="silu")
        self.time_text_embed = tte
        self.context_embedder = LoraLinear(cfg.joint_attention_dim, D)
        self.x_embedder = LoraLinear(cfg.in_channels, D)
        self.transformer_blocks = nn.ModuleList(
            [FluxDoubleBlock(D, cfg.num_attention_heads, cfg.attention_head_dim) for _ in range(cfg.num_layers)])
        self.single_transformer_blocks = nn.ModuleList(
            [FluxSingleBlock(D, cfg.num_attention_heads, cfg.attention_head_dim) for _ in range(cfg.num_single_layers)])
        self.norm_out = AdaLayerNormContinuous(D)
        self.proj_out = LoraLinear(D, cfg.patch_size ** 2 * (cfg.out_channels or cfg.in_channels))

    def forward(self, hidden_states, encoder_hidden_states=None, pooled_projections=None, timestep=None, img_ids=None,
                txt_ids=None, guidance=None, joint_attention_kwargs=None, return_dict=False, attention_mask=None):
        """The stock forward (transformer_flux.py:641-828) and, with `attention_mask` [B, T + L] and batched `img_ids` [B, L, 3], the
        custom multi-resolution forward (transformer_flux_custom.py:372-741): per-sample RoPE from each sample's valid ids with the
        identity rotation on padded positions (:494-553), padded image rows zeroed after x_embedder (:423-442), after every block
        (:645-661, 693-709) and in the output (:724-735), additive -inf key mask (:604-616)."""
        h = self.x_embedder(hidden_states)
        img_valid = add_mask = None
        if attention_mask is not None:
            T0 = txt_ids.shape[-2]
            m = attention_mask.to(h.device) > 0
            img_valid = m[:, T0:T0 + h.shape[1]]
            h = h.masked_fill(~img_valid.unsqueeze(-1), 0)
            add_mask = torch.zeros(m.shape[0], 1, 1, m.shape[1], dtype=h.dtype, device=h.device).masked_fill(~m[:, None, None, :], float("-inf"))
        t = timestep.to(h.dtype) * 1000
        tte = self.time_text_embed
        temb = tte.timestep_embedder(timestep_sinusoid(t, 256).to(pooled_projections.dtype))
        if guidance is not None:
            g = guidance.to(h.dtype) * 1000
            temb = temb + tte.guidance_embedder(timestep_sinusoid(g, 256).to(pooled_projections.dtype))
        temb = temb + tte.text_embedder(pooled_projections)
        enc = self.context_embedder(encoder_hidden_states)
        if img_ids.ndim == 3 and attention_mask is None:
            img_ids = img_ids[0]  # batched ids without a mask: shared layout (transformer_flux_custom.py:473-476)
        if txt_ids.ndim == 3:
            txt_ids = txt_ids[0]
        if img_ids.ndim == 3:
            cs, sn = [], []
            for b in range(img_ids.shape[0]):
                nv = int(img_valid[b].sum())
                c, s_ = flux_rope(torch.cat((txt_ids, img_ids[b, :nv]), dim=0), self.config.axes_dims_rope)
                pad = img_ids.shape[1] - nv
                cs.append(torch.cat([c, torch.ones(pad, c.shape[1], device=c.device)], 0))   # identity rotation on the padding
                sn.append(torch.cat([s_, torch.zeros(pad, c.shape[1], device=c.device)], 0))
            rope = (torch.stack(cs), torch.stack(sn))
        else:
            rope = flux_rope(torch.cat((txt_ids, img_ids), dim=0), self.config.axes_dims_rope)
        for blk in self.transformer_blocks:
            enc, h = blk(h, enc, temb, rope, add_mask)
            if img_valid is not None:
                h = h * img_valid.unsqueeze(-1)
        for blk in self.single_transformer_blocks:
            enc, h = blk(h, enc, temb, rope, add_mask)
            if img_valid is not None:
                h = h * img_valid.unsqueeze(-1)
        out = self.proj_out(self.norm_out(h, temb))
        if img_valid is not None:
            out = out.masked_fill(~img_valid.unsqueeze(-1), 0)
        return (out,)


# ----------------------------------------------------------------------------------------------------------------
# LoRA injection (base_trainer.py:929-941 -> peft LoraConfig(r, lora_alpha, init_lora_weights, target_modules))
# ----------------------------------------------------------------------------------------------------------------
DEFAULT_TARGETS = ("to_q", "to_k", "to_v", "to_out.0")  # data/config.py:315


def lora_targets(model: nn.Module, target_modules=DEFAULT_TARGETS) -> list[tuple[str, LoraLinear]]:
    """PEFT matching: a list matches by name suffix (`name == t or name.endswith('.'+t)`), a str is a full regex."""
    import re
    out = []
    for name, mod in model.named_modules():
        if not isinstance(mod, LoraLinear):
            continue
        if isinstance(target_modules, str):
            ok = re.fullmatch(target_modules, name) is not None
        else:
            ok = any(name == t or name.endswith("." + t) for t in target_modules)
        if ok:
            out.append((name, mod))
    return out


def add_lora_adapter(model: nn.Module, r: int, alpha: float, target_modules=DEFAULT_TARGETS, init="gaussian",
                     seed: int = 0, b_std: float = 0.0):
    g = torch.Generator().manual_seed(seed)
    for p in model.parameters():
        p.requires_grad_(False)
    for _, mod in lora_targets(model, target_modules):
        mod.add_adapter(r, alpha, init, g, b_std)
    for n, p in model.named_parameters():
        p.requires_grad_("lora" in n)  # qwen_image_edit_trainer.py:314-318
    return model


def init_synthetic_(model: nn.Module, seed: int = 1234, std: float = 0.02):
    """SURVEY.md §8d cfg 2: weights N(0, 0.02^2), biases 0, norm weights 1 (AdaLN linears non-zero so gates != 0)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for n, p in model.named_parameters():
            if "lora" in n:
                continue
            if n.endswith("bias"):
                p.zero_()
            elif p.ndim == 1:
                p.fill_(1.0)
            else:
                p.copy_(torch.randn(p.shape, generator=g, dtype=torch.float32) * std)
    return model


# ----------------------------------------------------------------------------------------------------------------
# training-step recipes
# ----------------------------------------------------------------------------------------------------------------
def qwen_img_shapes_latent(img_shapes_px, vae_scale=8, patch=2):
    """qwen_image_edit_trainer.py:557-577 convert_img_shapes_to_latent_space: (3,H,W) px -> (1,H/16,W/16)."""
    return [[(1, s[1] // vae_scale // patch, s[2] // vae_scale // patch) for s in sample] for sample in img_shapes_px]


def qwen_compute_loss(dit, image_latents, control_latents, prompt_embeds, prompt_embeds_mask, img_shapes, *, noise, u,
                      criterion=None):
    """qwen_image_edit_trainer.py:777-849 with `noise` and `u` (the CPU uniform draw) passed in so the recipe is
    deterministic: idx=(u*1000).long(); timesteps=linspace(1,1000,1000)[::-1][idx]; sigma=t/1000."""
    B = image_latents.shape[0]
    with torch.no_grad():
        idx = (u * 1000).long()
        sched_t = torch.linspace(1, 1000, 1000).flip(0)
        timesteps = sched_t[idx].to(image_latents.device)
        sigmas = (timesteps / 1000).to(image_latents.dtype).view(B, 1, 1)
        noisy = (1.0 - sigmas) * image_latents + sigmas * noise
        packed = torch.cat([noisy, control_latents], dim=1)
        txt_seq_lens = prompt_embeds_mask.sum(dim=1).tolist()
    pred = dit(hidden_states=packed, timestep=timesteps / 1000, guidance=None,
               encoder_hidden_states_mask=prompt_embeds_mask, encoder_hidden_states=prompt_embeds,
               img_shapes=img_shapes, txt_seq_lens=txt_seq_lens, return_dict=False)[0]
    pred = pred[:, : image_latents.size(1)]
    weighting = torch.ones_like(sigmas)
    target = noise - image_latents
    if criterion is None:  # MseLoss weighted branch (mse_loss.py:72-82)
        loss = (weighting.float() * (pred.float() - target.float()) ** 2).reshape(B, -1).mean(1).mean()
    else:
        loss = criterion(model_pred=pred, target=target, weighting=weighting, attention_mask=None, edit_mask=None)
    return loss, pred


def flux_latent_image_ids(h2, w2, first=0.0):
    """flux_kontext_trainer.py:869-883 _prepare_latent_image_ids; ids [h2*w2, 3] = (first, row, col)."""
    ids = torch.zeros(h2, w2, 3)
    ids[..., 0] = first
    ids[..., 1] = ids[..., 1] + torch.arange(h2)[:, None]
    ids[..., 2] = ids[..., 2] + torch.arange(w2)[None, :]
    return ids.reshape(h2 * w2, 3)


def flux_compute_loss_shared(dit, image_latents, control_latents, pooled, prompt_embeds, text_ids, image_ids,
                             control_ids, *, noise, t):
    """flux_kontext_trainer.py:494-577: x_t=(1-t)x0+t*eps; model(timestep=t); F.mse_loss in the working dtype."""
    B = image_latents.shape[0]
    t_ = t.view(B, 1, 1).to(image_latents.dtype)
    noisy = (1.0 - t_) * image_latents + t_ * noise
    latent_in = torch.cat([noisy, control_latents], dim=1)
    ids = torch.cat([image_ids, control_ids], dim=0)
    guidance = torch.ones(B, device=image_latents.device) if dit.config.guidance_embeds else None
    pred = dit(hidden_states=latent_in, timestep=t, guidance=guidance, pooled_projections=pooled,
               encoder_hidden_states=prompt_embeds, txt_ids=text_ids, img_ids=ids, return_dict=False)[0]
    pred = pred[:, : image_latents.size(1)]
    target = noise - image_latents
    return F.mse_loss(pred, target), pred
