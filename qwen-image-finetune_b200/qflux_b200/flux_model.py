"""B200-native FLUX.1 (Kontext) MMDiT with fused-LoRA training step — drop-in for the FLUX trainers' `self.dit`.

Mirrors `FluxTransformer2DModel` (/root/reference/src/qflux/models/transformer_flux.py:557-828; the shared-resolution
trainer path loads diffusers' identical class, flux_kontext_loader.py:157-160; call site
/root/reference/src/qflux/trainer/flux_kontext_trainer.py:555-565): same forward kwargs, same state-dict key names.

Double-stream blocks (transformer_flux.py:439-523) reuse the Qwen block launch sequence of mmdit_base.py — AdaLayerNormZero has
the same (shift, scale, gate) x (msa, mlp) chunk order; differences: torch.nn.RMSNorm for q/k (single rounding) and RoPE
positions from `ids` applied on the joint sequence.  Single-stream blocks (transformer_flux.py:385-436) run on the same
stream-major rows with ONE weight set for both row groups; `proj_out(cat[attn, gelu(proj_mlp)])` is a single contraction
whose K loop is extended over the MLP activations (the same k-block extension mechanism that fuses LoRA), and its two
dgrads are summed by the `ADD` epilogue.
"""
from __future__ import annotations

from dataclasses import dataclass

import torch

from . import lib
from .mmdit_base import BF, DEFAULT_TARGETS, PAD, FusedMMDiTBase  # noqa: F401
from .rope import flux_rope_table


@dataclass
class FluxB200Config:
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

    def __getitem__(self, k):
        return getattr(self, k)


# `model.lora.target_modules` of the reference's FLUX-Kontext config (BASELINE configs[2]; /root/reference/configs/face_seg_flux_kontext_fp16.yaml:11):
# every block Linear, the AdaLN modulation linears and x_embedder
FLUX_KONTEXT_YAML_TARGETS = (
    r"(.*x_embedder|.*transformer_blocks\.[0-9]+\.(norm|norm1)\.linear|.*transformer_blocks\.[0-9]+\.attn\.(to_k|to_q|to_v|to_add_out)"
    r"|.*transformer_blocks\.[0-9]+\.attn\.to_out\.0|.*single_transformer_blocks\.[0-9]+\.attn\.to_out"
    r"|.*single_transformer_blocks\.[0-9]+\.(proj_mlp|proj_out)|.*(?<!single_)transformer_blocks\.[0-9]+\.ff\.net\.2"
    r"|.*(?<!single_)transformer_blocks\.[0-9]+\.ff\.net\.0\.proj|.*(?<!single_)transformer_blocks\.[0-9]+\.norm1_context\.linear"
    r"|.*(?<!single_)transformer_blocks\.[0-9]+\.ff_context\.net\.0\.proj|.*(?<!single_)transformer_blocks\.[0-9]+\.ff_context\.net\.2"
    r"|.*(?<!single_)transformer_blocks\.[0-9]+\.attn\.(to_add_out|add_k_proj|add_q_proj|add_v_proj))")

_SINGLE_LINEARS = {"attn.to_q": ("s_qkv", 0), "attn.to_k": ("s_qkv", 1), "attn.to_v": ("s_qkv", 2), "proj_mlp": ("s_mlp", 0),
                   "proj_out": ("s_out", 0)}


class FluxB200(FusedMMDiTBase):
    round_mid = False  # torch.nn.RMSNorm (transformer_flux.py:342-343): one rounding after the weight multiply
    _DOUBLE_LINEARS = {
        "attn.to_q": ("qkv", 0, 0), "attn.to_k": ("qkv", 0, 1), "attn.to_v": ("qkv", 0, 2),
        "attn.add_q_proj": ("qkv", 1, 0), "attn.add_k_proj": ("qkv", 1, 1), "attn.add_v_proj": ("qkv", 1, 2),
        "attn.to_out.0": ("out", 0, 0), "attn.to_add_out": ("out", 1, 0),
        "ff.net.0.proj": ("up", 0, 0), "ff_context.net.0.proj": ("up", 1, 0),
        "ff.net.2": ("down", 0, 0), "ff_context.net.2": ("down", 1, 0),
    }
    _ADALN = ("norm1.linear", "norm1_context.linear")
    _PER_SINGLE = ("s_mod_w", "s_mod_b", "s_qkv_w", "s_qkv_b", "s_mlp_w", "s_mlp_b", "s_out_w", "s_out_b", "s_qknorm_w")
    _NF4_KINDS = FusedMMDiTBase._NF4_KINDS + ("s_mod_w", "s_qkv_w", "s_mlp_w", "s_out_w")
    _SINGLE_MATS = {**{nm: grp + "_w" for nm, (grp, _) in _SINGLE_LINEARS.items()}, "norm.linear": "s_mod_w"}

    def __init__(self, cfg: FluxB200Config, device="cuda", _host_only: bool = False, frozen_weights="bf16", nf4_blocksize: int = 64):
        """frozen_weights / nf4_blocksize: as for QwenImageB200 (4-bit and float8-e4m3fn base checkpoints)."""
        super().__init__()
        self._init_common(device, _host_only, frozen_weights, nf4_blocksize)
        assert cfg.attention_head_dim == 128, "the sm_90a attention kernels are specialised for head_dim 128"
        self.config = cfg
        D = cfg.num_attention_heads * cfg.attention_head_dim
        self.D, self.H, self.J = D, cfg.num_attention_heads, cfg.joint_attention_dim
        self.L, self.Ls = cfg.num_layers, cfg.num_single_layers
        self.C_in = cfg.in_channels
        self.C_out = cfg.patch_size ** 2 * (cfg.out_channels or cfg.in_channels)
        self.Pp = cfg.pooled_projection_dim
        L, Ls, J = self.L, self.Ls, self.J
        z = lambda *s: torch.zeros(*s, device=self.dev, dtype=BF)
        f = self._frozen
        self.w = {
            "x_in_w": z(D, self.C_in), "x_in_b": z(D), "ctx_in_w": z(D, J), "ctx_in_b": z(D),
            "t1_w": z(D, 256), "t1_b": z(D), "t2_w": z(D, D), "t2_b": z(D),
            "g1_w": z(D, 256), "g1_b": z(D), "g2_w": z(D, D), "g2_b": z(D),
            "p1_w": z(D, self.Pp), "p1_b": z(D), "p2_w": z(D, D), "p2_b": z(D),
            "mod_w": f("mod_w", L, 2, 6 * D, D), "mod_b": z(L, 2, 6 * D),
            "qkv_w": f("qkv_w", L, 2, 3 * D, D), "qkv_b": z(L, 2, 3 * D),
            "out_w": f("out_w", L, 2, D, D), "out_b": z(L, 2, D),
            "up_w": f("up_w", L, 2, 4 * D, D), "up_b": z(L, 2, 4 * D),
            "down_w": f("down_w", L, 2, D, 4 * D), "down_b": z(L, 2, D),
            "qknorm_w": torch.ones(L, 4, 128, device=self.dev, dtype=BF),
            "s_mod_w": f("s_mod_w", Ls, 3 * D, D), "s_mod_b": z(Ls, 3 * D),
            "s_qkv_w": f("s_qkv_w", Ls, 3 * D, D), "s_qkv_b": z(Ls, 3 * D),
            "s_mlp_w": f("s_mlp_w", Ls, 4 * D, D), "s_mlp_b": z(Ls, 4 * D),
            "s_out_w": f("s_out_w", Ls, D, 5 * D), "s_out_b": z(Ls, D),
            "s_qknorm_w": torch.ones(Ls, 2, 128, device=self.dev, dtype=BF),
            "norm_out_w": z(2 * D, D), "norm_out_b": z(2 * D),
            "proj_out_w": z(self.C_out, D), "proj_out_b": z(self.C_out),
        }
        self._finish_frozen()

    def _wb(self, l, grp, s):
        if l < 0:
            return self.w[grp + "_w"], self.w[grp + "_b"]
        if grp.startswith("s_"):
            return self.w[grp + "_w"][l], self.w[grp + "_b"][l]
        return self.w[grp + "_w"][l, s], self.w[grp + "_b"][l, s]

    # ------------------------------------------------------------------------------------------------ names
    def _weight_views(self, store: bool = False) -> dict:
        (w, blocks), D, out = self._view_source(store), self.D, {}
        out["x_embedder.weight"], out["x_embedder.bias"] = w["x_in_w"], w["x_in_b"]
        out["context_embedder.weight"], out["context_embedder.bias"] = w["ctx_in_w"], w["ctx_in_b"]
        for pre, nm in (("t", "timestep_embedder"), ("p", "text_embedder")) + ((("g", "guidance_embedder"),) if self.config.guidance_embeds else ()):
            p = f"time_text_embed.{nm}."
            out[p + "linear_1.weight"], out[p + "linear_1.bias"] = w[pre + "1_w"], w[pre + "1_b"]
            out[p + "linear_2.weight"], out[p + "linear_2.bias"] = w[pre + "2_w"], w[pre + "2_b"]
        out["norm_out.linear.weight"], out["norm_out.linear.bias"] = w["norm_out_w"], w["norm_out_b"]
        out["proj_out.weight"], out["proj_out.bias"] = w["proj_out_w"], w["proj_out_b"]
        self._double_weight_views(out, w, blocks)
        for l in range(self.Ls if blocks else 0):
            b = f"single_transformer_blocks.{l}."
            out[b + "norm.linear.weight"], out[b + "norm.linear.bias"] = w["s_mod_w"][l], w["s_mod_b"][l]
            out[b + "attn.norm_q.weight"], out[b + "attn.norm_k.weight"] = w["s_qknorm_w"][l, 0], w["s_qknorm_w"][l, 1]
            for nm, (grp, slot) in _SINGLE_LINEARS.items():
                W, Bv = w[grp + "_w"][l], w[grp + "_b"][l]
                if grp == "s_qkv":
                    W, Bv = W[slot * D:(slot + 1) * D], Bv[slot * D:(slot + 1) * D]
                out[b + nm + ".weight"], out[b + nm + ".bias"] = W, Bv
        return out

    def _linear_table(self) -> dict:
        D = self.D
        dims = {"s_qkv": (D, D, 3), "s_mlp": (D, 4 * D, 1), "s_out": (5 * D, D, 1)}
        t = super()._linear_table()
        for l in range(self.Ls):
            for nm, (grp, slot) in _SINGLE_LINEARS.items():
                d_in, d_out, n = dims[grp]
                t[f"single_transformer_blocks.{l}.{nm}"] = ((l, grp), (0, 1), slot, d_in, d_out, n)
        return t

    def _mod_table(self) -> dict:
        t = super()._mod_table()
        for l in range(self.Ls):
            t[f"single_transformer_blocks.{l}.norm.linear"] = ("sgl", l, 3)
        return t

    def _embed_table(self) -> dict:
        return {"x_embedder": ("x_in", 0, self.C_in), "context_embedder": ("ctx_in", 1, self.J)}

    # ------------------------------------------------------------------------------------------------ workspace
    def _workspace(self, B, T, Limg, train: bool):
        D = self.D
        extra = [(k, (B, 256)) for k in ("sin", "gsin")] + [(k, (B, D)) for k in ("e1", "temb", "gemb", "pemb")]
        extra += [("mods", (B, self.L * 2 * 6 * D)), ("smods", (B, max(self.Ls, 1) * 3 * D)), ("fmod", (B, 2 * D))]
        det = train and torch.are_deterministic_algorithms_enabled()  # read on every forward: selects the fixed-order backward
        return self._get_workspace((B, T, Limg, train, det),
                                   lambda: self._alloc_common({}, B, T, Limg, train, self.L, self.Ls, extra=extra, det=det))

    # ------------------------------------------------------------------------------------------------ single block
    def _single_fwd(self, ws, l, Xin, Xout, save, recompute=False):
        """recompute: as in `_double_fwd` — proj_out only runs when its un-gated output feeds the AdaLN-LoRA gate gradient."""
        D, w = self.D, self.w
        T, Mt = ws["T"], ws["Mt"]
        st, qkv, O, h, u = save["stats"], save["qkv"], save["O"], save["h"], save["u"]
        self._ln_fwd2(ws, Xin, ws["xm"], self._smod(ws, l, 0), self._smod(ws, l, 1), st[0], st[1])
        self._grouped(ws, l, "s_qkv", ws["xm"], qkv, 3 * D, D, lib.EPI_BIAS)
        self._grouped(ws, l, "s_mlp", ws["xm"], h, 4 * D, D, lib.EPI_GELU, out2=u)
        qn = w["s_qknorm_w"][l]
        lib.qk_norm_rope_fwd_pair(qkv, (qn[0], qn[1], T, 0), (qn[0], qn[1], ws["Limg"], T), Mt, ws["rope"], ws["Q"], ws["K"], ws["V"],
                                  round_mid=False)
        lib.attn_fwd(ws["Q"], ws["K"], ws["V"], O[:Mt], O[Mt:], T, save["lse"], kv_len=ws.get("kv_len"), txt_len=ws.get("txt_len"))
        # x = x + gate * proj_out(cat[attn, gelu(mlp)]): attention wrote columns [0, D) and the GELU epilogue [D, 5D) of save["cat"]
        if not recompute or self._keeps_gate_out(l, "sgl"):
            self._grouped(ws, l, "s_out", save["cat"], Xout, D, 5 * D, lib.EPI_RESID_GATE, resid=Xin, gate=self._smod(ws, l, 2),
                          out2=save.get("y_out"))

    def _single_bwd(self, ws, l, Xin, dX, dXn, save, prev_gate):
        D, w = self.D, self.w
        st, qkv, O, u = save["stats"], save["qkv"], save["O"], save["u"]
        Wo = w["s_out_w"][l]
        dsm = lambda j: self._dmod(ws, "sgl", l, j)  # d(shift, scale, gate): ONE vector per sample for text and image rows alike
        if dsm(2) is not None:
            for s in (0, 1):
                self._mod_grad(ws, self._rows(ws, dX, s), self._rpb(ws, s), m=self._rows(ws, save["y_out"], s), prod_out=dsm(2))
        # d[attn | mlp] = dY . W_out (+ U . A_lora)   (dY = dX * gate is already in ws['dY']); the two column ranges of the
        # concatenated input go to different consumers (attention backward / GELU backward), so they are two contractions
        pa, pm = [], []
        lbs = self._lora_bwd_pair(ws, l, "s_out", ws["dY"], save["cat"], D)
        for s in (0, 1):
            dYs = self._rows(ws, ws["dY"], s)
            lb = lbs[s]
            ka = dict(A2=lb[0], B2=lb[1][:, :D], kb2=lb[2]) if lb is not None else {}
            km = dict(A2=lb[0], B2=lb[1][:, D:], kb2=lb[2]) if lb is not None else {}
            pa.append((dYs, Wo[:, :D], ka))
            pm.append(lib.gemm_problem(dYs, Wo[:, D:], self._rows(ws, ws["dbig"], s), aux=self._rows(ws, u, s),
                                       row_bands=self._bands(ws, s), **km))
        self._dgrad_attn_out(ws, pa, O, D, D)  # d attn: straight into the attention backward's layout (+ delta)
        lib.gemm(pm, 4 * D, D, trans_b=True, epilogue=lib.EPI_DGELU)
        self._attn_bwd_core(ws, qkv, O, save["lse"], lambda s: (w["s_qknorm_w"][l, 0], w["s_qknorm_w"][l, 1]))
        if self._site(l, "s_qkv", 0) or self._site(l, "s_mlp", 0):  # LoRA input = modulated norm output (recomputed)
            self._ln_fwd2(ws, Xin, ws["xm"], self._smod(ws, l, 0), self._smod(ws, l, 1))
        self._dgrad_grouped(ws, l, "s_qkv", ws["dqkv"], ws["dxm"], D, 3 * D, D, ws["xm"])
        self._dgrad_grouped(ws, l, "s_mlp", ws["dbig"], ws["dxm"], D, 4 * D, 4 * D, ws["xm"], epilogue=lib.EPI_ADD, resid=ws["dxm"])
        for s in (0, 1):
            if dsm(0) is not None:
                self._mod_grad(ws, self._rows(ws, ws["dxm"], s), self._rpb(ws, s), sum_out=dsm(0), m=self._rows(ws, Xin, s),
                               prod_out=dsm(1), mean=self._rows(ws, st[0], s), rstd=self._rows(ws, st[1], s))
        self._ln_bwd2(ws, ws["dxm"], Xin, st[0], st[1], self._smod(ws, l, 1), dXn, dres=dX, gate=prev_gate, dx_gated=ws["dY"])

    # ------------------------------------------------------------------------------------------------ forward
    def _mlp2(self, x, pre, out, tmp):
        """linear_2(silu(linear_1(x))) on [B, *] conditioning vectors."""
        w = self.w
        lib.gemv_act(x, w[pre + "1_w"], w[pre + "1_b"], tmp, act=0)
        lib.gemv_act(tmp, w[pre + "2_w"], w[pre + "2_b"], out, act=1)

    def _forward_impl(self, hidden_states, encoder_hidden_states, pooled_projections, timestep, img_ids, txt_ids, guidance,
                      kv_len=None, train: bool = False, valid_rows=None):
        """img_ids [L, 3] (shared) or [B, L, 3] together with kv_len (int32 [B] on the device: T + valid image tokens) for a
        pad-to-max multi-resolution batch — per-sample RoPE tables and key masks (transformer_flux_custom.py:494-616)."""
        lib.require_cuda(hidden_states, encoder_hidden_states, pooled_projections, timestep, kv_len)
        B, Limg, _ = hidden_states.shape
        T = encoder_hidden_states.shape[1]
        D, L, Ls, w = self.D, self.L, self.Ls, self.w
        ws = self._workspace(B, T, Limg, train)
        self._fwd_gen += 1
        Mt = ws["Mt"]
        if txt_ids.ndim == 3:
            txt_ids = txt_ids[0]
        if img_ids.ndim == 3 and kv_len is None:
            img_ids = img_ids[0]  # batched ids without a mask: every sample has the same layout (transformer_flux_custom.py:473-476)
        # The table is rebuilt on every call (a few small device kernels, no host sync): the ids are data, and a cache keyed on the
        # tensor's address goes stale when the allocator hands the same block to the next batch's ids.
        ti, ii = txt_ids.to(self.dev), img_ids.to(self.dev)
        if ii.ndim == 3:  # zero-padded ids give position 0 on every axis = the identity rotation the reference pads with (:538-553)
            ws["rope"] = torch.stack([flux_rope_table(torch.cat((ti, ii[b]), dim=0), self.config.axes_dims_rope)
                                      for b in range(B)]).contiguous()
        else:
            ws["rope"] = flux_rope_table(torch.cat((ti, ii), dim=0), self.config.axes_dims_rope)
        ws["kv_len"] = kv_len
        self._plan_bands(ws, valid_rows if kv_len is not None else None)  # host copy of kv_len - T (None: every row is computed)
        assert ws["rope"].shape[-3] == ws["S"]
        X0 = ws["X"][0]
        # --- conditioning: temb = MLP_t(sin(1000 t)) [+ MLP_g(sin(1000 g))] + MLP_p(pooled)   (bf16 products, like the model)
        t32 = (timestep.to(BF) * 1000).float().contiguous()
        lib.timestep_sinusoid(t32, 1.0, ws["sin"])
        self._mlp2(ws["sin"], "t", ws["temb"], ws["e1"])
        if guidance is not None and self.config.guidance_embeds:
            g32 = (guidance.to(BF) * 1000).float().contiguous()
            lib.timestep_sinusoid(g32, 1.0, ws["gsin"])
            self._mlp2(ws["gsin"], "g", ws["gemb"], ws["e1"])
            lib.add_bf16(ws["temb"], ws["gemb"], ws["temb"])
        self._mlp2(pooled_projections.to(BF).contiguous(), "p", ws["pemb"], ws["e1"])
        lib.add_bf16(ws["temb"], ws["pemb"], ws["temb"])
        if self._blk_rings is None:  # all modulation linears of a kind in one launch; ringed weights produce them block by block
            lib.gemv_act(ws["temb"], w["mod_w"].view(L * 2 * 6 * D, D), w["mod_b"].view(-1), ws["mods"], act=1)
            if Ls:
                lib.gemv_act(ws["temb"], w["s_mod_w"].view(Ls * 3 * D, D), w["s_mod_b"].view(-1), ws["smods"], act=1)
            self._mod_lora_fwd(ws, ws["temb"])
        lib.gemv_act(ws["temb"], w["norm_out_w"], w["norm_out_b"], ws["fmod"], act=1)
        # --- embedders
        self._embed_fwd(ws, "x_in", 0, hidden_states.to(BF).reshape(B * Limg, self.C_in), X0[Mt:])
        self._embed_fwd(ws, "ctx_in", 1, encoder_hidden_states.to(BF).reshape(Mt, self.J), X0[:Mt])
        return self._blocks_and_head_fwd(ws, train)

    # ------------------------------------------------------------------------------------------------ public API
    def forward(self, hidden_states, encoder_hidden_states=None, pooled_projections=None, timestep=None, img_ids=None,
                txt_ids=None, guidance=None, joint_attention_kwargs=None, return_dict=False, attention_mask=None):
        """Padded image rows of a pad-to-max batch (`attention_mask`) come back as exact zeros (transformer_flux_custom.py:724-735)."""
        def make_args():
            kv_len, ids = None, img_ids
            if attention_mask is not None:  # [B, T + L] validity mask of a pad-to-max batch (prefix-valid per sample, tools.py:319-396)
                kv_len = attention_mask.to(self.dev).sum(dim=1).to(torch.int32)
                if ids.ndim == 2:
                    ids = ids[None].expand(hidden_states.shape[0], -1, -1)
            return (hidden_states, encoder_hidden_states, pooled_projections, timestep, ids, txt_ids, guidance, kv_len)
        return self._forward_tail(make_args)
