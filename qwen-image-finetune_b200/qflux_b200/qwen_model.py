"""B200-native Qwen-Image MMDiT with fused-LoRA training step — the drop-in for `trainer.dit`.

Mirrors the interface of the reference's `QwenImageTransformer2DModel`
(/root/reference/src/qflux/models/transformer_qwenimage.py:497-672; called at
/root/reference/src/qflux/trainer/qwen_image_edit_trainer.py:827-836): same forward kwargs, same state-dict key
names (diffusers + PEFT `base_layer` / `lora_A.default` / `lora_B.default`), LoRA A/B exposed as nn.Parameters whose
names contain "lora".  Every FLOP runs in libqfx_b200.so (hand-written sm_90a kernels); this file only sequences the
launches and owns the HBM layout (see mmdit_base.py / DESIGN.md §3):

  * frozen weights live in layer-stacked fused tensors (q|k|v concatenated per stream, both streams adjacent) so one
    grouped wgmma GEMM serves the image and text stream of a block;
  * LoRA factors live zero-padded to 64 rows/cols so they enter the K loop of the base GEMM as one extra k-block;
  * activations needed by the backward are kept in HBM: block inputs, LayerNorm statistics, pre-norm q|k|v, attention output +
    logsumexp, mid residual, MLP pre-activation.  On an 80 GB H100 they are what limits the batch, so the blocks whose saved
    tensors do not fit keep only their input and are re-run right before their backward (`activation_plan`, DESIGN.md §3).

No CPU path, no eager-PyTorch fallback: every op raises if the tensors are not on a CUDA device.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch

from . import lib
from .mmdit_base import BF, DEFAULT_TARGETS, PAD, FusedMMDiTBase  # noqa: F401
from .rope import qwen_rope_table


@dataclass
class QwenB200Config:
    patch_size: int = 2
    in_channels: int = 64
    out_channels: int = 16
    num_layers: int = 60
    attention_head_dim: int = 128
    num_attention_heads: int = 24
    joint_attention_dim: int = 3584
    guidance_embeds: bool = False
    axes_dims_rope: tuple = (16, 56, 56)

    def __getitem__(self, k):
        return getattr(self, k)


class _QwenPosEmbed:
    """`dit.pos_embed(img_shapes, txt_seq_lens, device=)` as the reference's trainer calls it for per-sample tables
    (/root/reference/src/qflux/trainer/qwen_image_edit_trainer.py:734; QwenEmbedRope.forward, transformer_qwenimage.py:197-235):
    returns (vid_freqs [sum f*h*w, 64], txt_freqs [max(txt_seq_lens), 64]) as complex64, from the same table the kernels use."""

    def __init__(self, axes_dim, theta=10000):
        self.axes_dim, self.theta = tuple(axes_dim), theta

    def __call__(self, video_fhw, txt_seq_lens, device=None):
        if isinstance(video_fhw, list) and video_fhw and isinstance(video_fhw[0], (list,)):
            video_fhw = video_fhw[0]  # only the first sample's shapes are used in shared mode (:206-207)
        if not isinstance(video_fhw, list):
            video_fhw = [video_fhw]
        T = int(max(txt_seq_lens)) if isinstance(txt_seq_lens, (list, tuple)) else int(txt_seq_lens)
        tab = qwen_rope_table([tuple(s) for s in video_fhw], T, self.axes_dim, float(self.theta))
        cis = torch.complex(tab[..., 0], tab[..., 1])
        if device is not None:
            cis = cis.to(device)
        return cis[T:], cis[:T]

    forward = __call__


class QwenImageB200(FusedMMDiTBase):
    round_mid = True
    _DOUBLE_LINEARS = {
        "attn.to_q": ("qkv", 0, 0), "attn.to_k": ("qkv", 0, 1), "attn.to_v": ("qkv", 0, 2),
        "attn.add_q_proj": ("qkv", 1, 0), "attn.add_k_proj": ("qkv", 1, 1), "attn.add_v_proj": ("qkv", 1, 2),
        "attn.to_out.0": ("out", 0, 0), "attn.to_add_out": ("out", 1, 0),
        "img_mlp.net.0.proj": ("up", 0, 0), "txt_mlp.net.0.proj": ("up", 1, 0),
        "img_mlp.net.2": ("down", 0, 0), "txt_mlp.net.2": ("down", 1, 0),
    }
    _ADALN = ("img_mod.1", "txt_mod.1")

    def __init__(self, cfg: QwenB200Config, device="cuda", _host_only: bool = False):
        """`_host_only=True` (tests of the naming / LoRA-registry logic) allocates on `device` without requiring CUDA;
        every compute entry point still raises on non-CUDA tensors."""
        super().__init__()
        self._init_common(device, _host_only)
        assert cfg.attention_head_dim == 128, "the sm_90a attention kernels are specialised for head_dim 128"
        self.config = cfg
        # Multi-resolution batches with PADDED TEXT: "aligned" rotates a sample's image tokens where they sit ([T, T + L_b)), which makes
        # a padded batch equal the per-sample runs; "reference" reproduces transformer_qwen_custom.py:199-208, which lays the image table
        # down right after the sample's un-padded text length.  The two agree when no text is padded (DESIGN.md §2).
        self.rope_placement = "aligned"
        self.pos_embed = _QwenPosEmbed(cfg.axes_dims_rope)
        D = cfg.num_attention_heads * cfg.attention_head_dim
        self.D, self.H, self.L, self.J = D, cfg.num_attention_heads, cfg.num_layers, cfg.joint_attention_dim
        self.C_in, self.C_out = cfg.in_channels, cfg.patch_size ** 2 * cfg.out_channels
        L, J = self.L, self.J
        z = lambda *s: torch.zeros(*s, device=self.dev, dtype=BF)
        # frozen weights (plain tensors, not Parameters: they never receive gradients on this path)
        self.w = {
            "img_in_w": z(D, self.C_in), "img_in_b": z(D), "txt_norm_w": torch.ones(J, device=self.dev, dtype=BF),
            "txt_in_w": z(D, J), "txt_in_b": z(D),
            "t1_w": z(D, 256), "t1_b": z(D), "t2_w": z(D, D), "t2_b": z(D),
            "mod_w": z(L, 2, 6 * D, D), "mod_b": z(L, 2, 6 * D),
            "qkv_w": z(L, 2, 3 * D, D), "qkv_b": z(L, 2, 3 * D),
            "out_w": z(L, 2, D, D), "out_b": z(L, 2, D),
            "up_w": z(L, 2, 4 * D, D), "up_b": z(L, 2, 4 * D),
            "down_w": z(L, 2, D, 4 * D), "down_b": z(L, 2, D),
            "qknorm_w": torch.ones(L, 4, 128, device=self.dev, dtype=BF),
            "norm_out_w": z(2 * D, D), "norm_out_b": z(2 * D),
            "proj_out_w": z(self.C_out, D), "proj_out_b": z(self.C_out),
        }

    # ------------------------------------------------------------------------------------------------ names
    def _weight_views(self) -> dict:
        w, out = self.w, {}
        out["img_in.weight"], out["img_in.bias"] = w["img_in_w"], w["img_in_b"]
        out["txt_norm.weight"] = w["txt_norm_w"]
        out["txt_in.weight"], out["txt_in.bias"] = w["txt_in_w"], w["txt_in_b"]
        p = "time_text_embed.timestep_embedder."
        out[p + "linear_1.weight"], out[p + "linear_1.bias"] = w["t1_w"], w["t1_b"]
        out[p + "linear_2.weight"], out[p + "linear_2.bias"] = w["t2_w"], w["t2_b"]
        out["norm_out.linear.weight"], out["norm_out.linear.bias"] = w["norm_out_w"], w["norm_out_b"]
        out["proj_out.weight"], out["proj_out.bias"] = w["proj_out_w"], w["proj_out_b"]
        return self._double_weight_views(out)

    def _embed_table(self) -> dict:
        return {"img_in": ("img_in", 0, self.C_in), "txt_in": ("txt_in", 1, self.J)}

    # ------------------------------------------------------------------------------------------------ workspace
    def _workspace(self, B, T, Limg, train: bool):
        D = self.D
        extra = [("sin", (B, 256)), ("t1", (B, D)), ("temb", (B, D)), ("mods", (B, self.L * 2 * 6 * D)), ("fmod", (B, 2 * D)),
                 ("txt_n", (B * T, self.J))]
        return self._get_workspace((B, T, Limg, train), lambda: self._alloc_common({}, B, T, Limg, train, self.L, extra=extra))

    def _rope(self, img_shapes, T):
        key = (tuple(tuple(s) for s in img_shapes), T)
        if key not in self._rope_cache:
            self._rope_cache[key] = qwen_rope_table(img_shapes, T, self.config.axes_dims_rope).to(self.dev)
        return self._rope_cache[key]

    # ------------------------------------------------------------------------------------------------ forward
    def _rope_multi(self, img_shapes, T, Limg, txt_lens=None):
        """Per-sample tables [B, T+Limg, 64, 2] for a pad-to-max multi-resolution batch; padded rows get the identity rotation
        (cos 1, sin 0 — transformer_flux_custom.py:148-154), their keys are masked anyway.  Returns (table, kv_len int32 [B]).
        txt_lens (host ints, `rope_placement="reference"` only): sample b's table is built for ITS text length and laid down from joint
        position 0 — text angles on [0, n_b), image angles on [n_b, n_b + L_b) — which is where the reference's
        `_apply_rope_per_sample` puts them (transformer_qwen_custom.py:199-208), text padding or not."""
        key = ("multi", tuple(tuple(tuple(s) for s in sh) for sh in img_shapes), T, Limg, None if txt_lens is None else tuple(txt_lens))
        if key not in self._rope_cache:
            if len(self._rope_cache) >= 64:  # bucketed multi-resolution training meets a bounded set of shape combinations; stay bounded anyway
                self._rope_cache.pop(next(iter(self._rope_cache)))
            tabs, lens = [], []
            for b, sh in enumerate(img_shapes):
                t = qwen_rope_table(sh, T if txt_lens is None else int(txt_lens[b]), self.config.axes_dims_rope)
                pad = torch.zeros(T + Limg - t.shape[0], t.shape[1], 2)
                pad[..., 0] = 1.0
                tabs.append(torch.cat([t, pad], 0))
                lens.append(T + sum(f * h * w for f, h, w in sh))  # keys live at their joint positions whatever the rotation placement
            self._rope_cache[key] = (torch.stack(tabs).contiguous().to(self.dev),
                                     torch.tensor(lens, dtype=torch.int32).to(self.dev))
        return self._rope_cache[key]

    def _forward_impl(self, hidden_states, encoder_hidden_states, timestep, img_shapes, txt_len=None, txt_seq_lens=None, *,
                      train: bool = False):
        """img_shapes: one list of (frame, h, w) per sample.  When the samples differ (multi-resolution, pad-to-max) every
        sample gets its own RoPE table and key mask (transformer_qwen_custom.py:444-553); `txt_len` (int32 [B] on the device)
        additionally masks text padding; `txt_seq_lens` (host ints) selects the reference's RoPE placement (see _rope_multi)."""
        lib.require_cuda(hidden_states, encoder_hidden_states, timestep, txt_len)
        B, Limg, _ = hidden_states.shape
        T = encoder_hidden_states.shape[1]
        D, L, w = self.D, self.L, self.w
        ws = self._workspace(B, T, Limg, train)
        self._fwd_gen += 1
        Mt = ws["Mt"]
        nested = isinstance(img_shapes[0], (list, tuple)) and isinstance(img_shapes[0][0], (list, tuple))
        per_sample = [list(map(tuple, sh)) for sh in img_shapes] if nested else [list(map(tuple, img_shapes))] * B
        if any(sh != per_sample[0] for sh in per_sample):
            assert len(per_sample) == B
            ws["rope"], ws["kv_len"] = self._rope_multi(per_sample, T, Limg, txt_seq_lens)
            self._plan_bands(ws, [sum(f * h * w for f, h, w in sh) for sh in per_sample])
        else:
            self._plan_bands(ws, None)
            rope = self._rope(per_sample[0], T)
            assert rope.shape[0] == ws["S"], f"img_shapes {per_sample[0]} do not add up to {Limg} image tokens"
            ws["rope"], ws["kv_len"] = rope, None
        ws["txt_len"] = txt_len
        X0 = ws["X"][0]
        # --- conditioning: sigma (bf16-rounded, transformer_qwenimage.py:624) -> sinusoid -> MLP -> all modulation vectors
        t32 = timestep.to(BF).float().contiguous()
        lib.timestep_sinusoid(t32, 1000.0, ws["sin"])
        lib.gemv_act(ws["sin"], w["t1_w"], w["t1_b"], ws["t1"], act=0)
        lib.gemv_act(ws["t1"], w["t2_w"], w["t2_b"], ws["temb"], act=1)
        if self._sharded is None:  # all 2L modulation linears in one launch; sharded weights produce them block by block
            lib.gemv_act(ws["temb"], w["mod_w"].view(L * 2 * 6 * D, D), w["mod_b"].view(-1), ws["mods"], act=1)
            self._mod_lora_fwd(ws, ws["temb"])
        lib.gemv_act(ws["temb"], w["norm_out_w"], w["norm_out_b"], ws["fmod"], act=1)
        # --- embedders
        hs = hidden_states.to(BF).reshape(B * Limg, self.C_in)
        self._embed_fwd(ws, "img_in", 0, hs, X0[Mt:])
        lib.rmsnorm_rows(encoder_hidden_states.to(BF).reshape(Mt, self.J), w["txt_norm_w"], ws["txt_n"])
        self._embed_fwd(ws, "txt_in", 1, ws["txt_n"], X0[:Mt])
        return self._blocks_and_head_fwd(ws, train)

    # ------------------------------------------------------------------------------------------------ public API
    def forward(self, hidden_states, encoder_hidden_states=None, encoder_hidden_states_mask=None, timestep=None,
                img_shapes=None, txt_seq_lens=None, guidance=None, attention_kwargs=None, return_dict=False):
        """Same signature as the reference model.  With grad enabled and an adapter attached the result carries
        autograd history to the LoRA parameters (custom Function around the fused backward)."""
        def make_args():
            nested = isinstance(img_shapes[0], (list, tuple)) and isinstance(img_shapes[0][0], (list, tuple))
            multi = nested and any(list(map(tuple, sh)) != list(map(tuple, img_shapes[0])) for sh in img_shapes)
            txt_len = None
            if multi and encoder_hidden_states_mask is not None:  # the mask is only honoured in multi-resolution mode (like the reference)
                txt_len = encoder_hidden_states_mask.to(self.dev).sum(dim=1).to(torch.int32)
            args = (hidden_states, encoder_hidden_states, timestep, img_shapes)
            if multi:
                args = args + (txt_len,)
                if self.rope_placement == "reference":
                    if txt_seq_lens is None:
                        raise ValueError("rope_placement='reference' needs txt_seq_lens (one text length per sample), as the reference's forward takes it")
                    args = args + (tuple(int(n) for n in txt_seq_lens),)
            return args
        return self._forward_tail(make_args)
