"""Host-side logic of the fused model (launch sequencing, operand wiring, LoRA registry, gradient offsets) on CPU:
`qflux_b200.lib` is replaced by the plain-PyTorch emulation in tests/emu_lib.py and the result is compared with the oracle.
(The CUDA kernels themselves are covered by the `-m gpu` tests.)"""
import pytest
import torch

import emu_lib
from oracle import mmdit_oracle as mo


@pytest.fixture()
def emu():
    from qflux_b200 import lib
    restore = emu_lib.install(lib)
    yield lib
    restore()


def _pair(H, L, J, r, targets):
    from qflux_b200.qwen_model import QwenB200Config, QwenImageB200
    cfg = mo.QwenConfig(num_layers=L, attention_head_dim=128, num_attention_heads=H, joint_attention_dim=J)
    orc = mo.init_synthetic_(mo.QwenImageOracle(cfg), std=0.05)
    g = torch.Generator().manual_seed(99)
    with torch.no_grad():
        for n, p in orc.named_parameters():
            if n.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.02)
            elif p.ndim == 1:
                p.copy_(1 + torch.randn(p.shape, generator=g) * 0.1)
    if r:
        mo.add_lora_adapter(orc, r=r, alpha=2 * r, target_modules=targets, b_std=0.05)
    with torch.no_grad():
        for p in orc.parameters():
            p.copy_(p.bfloat16().float())
    m = QwenImageB200(QwenB200Config(num_layers=L, num_attention_heads=H, joint_attention_dim=J), device="cpu", _host_only=True)
    if r:
        m.add_adapter(r, 2 * r, target_modules=targets)
    missing, unexpected = m.load_state_dict(orc.state_dict(), strict=True)
    assert not missing and not unexpected
    return orc, m


def _inputs(B, hw, T, J):
    g = torch.Generator().manual_seed(0)
    rn = lambda *s: torch.randn(*s, generator=g).bfloat16()
    return dict(image_latents=rn(B, hw * hw, 64), control_latents=rn(B, hw * hw, 64), prompt_embeds=rn(B, T, J) * 3,
                prompt_embeds_mask=torch.ones(B, T, dtype=torch.int64), img_shapes=[[(1, hw, hw), (1, hw, hw)]] * B,
                noise=rn(B, hw * hw, 64), u=torch.tensor([0.5, 0.25, 0.125][:B]))  # sigma = .5, .75, .875: exact in bf16 (the model rounds t to bf16, :624)


@pytest.mark.parametrize("targets,r", [(("to_q", "to_k", "to_v", "to_out.0"), 4),
                                       (("to_q", "to_v", "add_k_proj", "to_add_out", "net.0.proj"), 8),
                                       (("to_k", "img_mlp.net.2", "txt_mlp.net.0.proj", "txt_mlp.net.2"), 4),
                                       (("to_q", "img_mod.1", "txt_mod.1", "img_in", "txt_in"), 4)])
def test_step_matches_oracle_on_cpu(emu, targets, r):
    from qflux_b200.train_step import QwenImageEditStep
    orc, m = _pair(2, 2, 128, r, targets)
    x = _inputs(2, 4, 24, 128)
    xf = {k: (v.float() if torch.is_tensor(v) and v.is_floating_point() and k != "u" else v) for k, v in x.items()}
    loss_o, pred_o = mo.qwen_compute_loss(orc, **xf)
    loss_o.backward()
    step = QwenImageEditStep(m)
    emb = {k: x[k] for k in ("image_latents", "control_latents", "prompt_embeds", "img_shapes")}
    loss_b = step.compute_loss(emb, noise=x["noise"], u=x["u"])
    pred_b = m._ws["pred"].view(2, -1, 64)[:, :16].float().clone()
    loss_b.backward()
    rel = ((pred_b - pred_o).norm() / pred_o.norm()).item()
    assert rel < 1e-2, rel                                  # bf16 storage vs fp32 oracle (BASELINE.md §3)
    assert abs(loss_b.item() - loss_o.item()) < 1e-2
    go = {n: (p.grad if p.grad is not None else torch.zeros_like(p)) for n, p in orc.named_parameters() if p.requires_grad}
    gb = {n: p.grad.float() for n, p in m.named_parameters()}
    assert set(go) == set(gb)
    num = sum(((gb[n] - go[n]) ** 2).sum() for n in go)
    den = sum((go[n] ** 2).sum() for n in go)
    assert float((num / den).sqrt()) < 2e-2
    # the no-autograd fast path produces the same gradients, clipped to max_grad_norm = 1
    step.train_step(emb, noise=x["noise"], u=x["u"])
    gnorm = float(den.sqrt())
    for n, p in m.named_parameters():
        ref = go[n] * min(1.0, 1.0 / (gnorm + 1e-6))
        if ref.abs().max() > 0:
            assert ((p.grad.float() - ref).norm() / ref.norm()).item() < 3e-2, n


def test_module_forward_signature_no_grad(emu):
    orc, m = _pair(2, 1, 128, 0, None)
    x = _inputs(2, 4, 24, 128)
    packed = torch.cat([x["image_latents"], x["control_latents"]], 1)
    t = torch.tensor([0.75, 0.25])
    with torch.no_grad():
        po = orc(hidden_states=packed.float(), timestep=t, encoder_hidden_states=x["prompt_embeds"].float(),
                 encoder_hidden_states_mask=x["prompt_embeds_mask"], img_shapes=x["img_shapes"], txt_seq_lens=[24, 24])[0]
        pb = m(hidden_states=packed, timestep=t, guidance=None, encoder_hidden_states_mask=x["prompt_embeds_mask"],
               encoder_hidden_states=x["prompt_embeds"], img_shapes=x["img_shapes"], txt_seq_lens=[24, 24], return_dict=False)[0]
    assert pb.shape == po.shape
    assert ((pb.float() - po).norm() / po.norm()).item() < 1e-2


def test_module_forward_autograd_bridge(emu):
    """`dit(...)` under grad mode carries autograd history to the LoRA parameters (drop-in for arbitrary losses)."""
    orc, m = _pair(2, 1, 128, 4, ("to_q", "to_k", "to_v", "to_out.0"))
    x = _inputs(1, 4, 24, 128)
    packed = torch.cat([x["image_latents"], x["control_latents"]], 1)
    t = torch.tensor([0.625])
    kw = dict(timestep=t, encoder_hidden_states_mask=x["prompt_embeds_mask"], img_shapes=x["img_shapes"], txt_seq_lens=[24])
    po = orc(hidden_states=packed.float(), encoder_hidden_states=x["prompt_embeds"].float(), **kw)[0]
    po.pow(2).mean().backward()
    pb = m(hidden_states=packed, encoder_hidden_states=x["prompt_embeds"], **kw)[0]
    pb.float().pow(2).mean().backward()
    go = {n: p.grad for n, p in orc.named_parameters() if p.requires_grad}
    num = sum(((p.grad.float() - go[n]) ** 2).sum() for n, p in m.named_parameters())
    den = sum((v ** 2).sum() for v in go.values())
    assert float((num / den).sqrt()) < 2e-2


def test_lora_registry_and_errors():
    from qflux_b200.qwen_model import QwenB200Config, QwenImageB200
    m = QwenImageB200(QwenB200Config(num_layers=2, num_attention_heads=2, joint_attention_dim=128), device="cpu", _host_only=True)
    with pytest.raises(NotImplementedError):
        m.add_adapter(4, 4, target_modules=r".*(norm_out\.linear|attn\.to_q)")
    m = QwenImageB200(QwenB200Config(num_layers=2, num_attention_heads=2, joint_attention_dim=128), device="cpu", _host_only=True)
    m.add_adapter(16, 16)
    names = [n for n, _ in m.named_parameters()]
    assert len(names) == 2 * 4 * 2 and all("lora" in n for n in names)
    assert m.G32.numel() == sum(p.numel() for p in m.parameters())
    # padded storage stays zero outside the adapter's rank
    site = m.sites[(0, "qkv", 0)]
    assert site.A_pad[16:64].abs().sum() == 0 and site.B_pad[:, 16:].abs().sum() == 0
    # ops refuse CPU tensors (no fallback)
    from qflux_b200 import lib
    with pytest.raises(lib.QfxError):
        lib.rmsnorm_rows(torch.zeros(8, 64, dtype=torch.bfloat16), torch.ones(64, dtype=torch.bfloat16), torch.zeros(8, 64, dtype=torch.bfloat16))


# ------------------------------------------------------------------------------------------------------------------ FLUX
# target_modules of BASELINE config 3 (/root/reference/configs/face_seg_flux_kontext_fp16.yaml:11): every Linear of every block incl. the
# AdaLN modulation linears, plus x_embedder
FLUX_YAML_TARGETS = (r"(.*x_embedder|.*transformer_blocks\.[0-9]+\.(norm|norm1)\.linear|.*transformer_blocks\.[0-9]+\.attn\.(to_k|to_q|to_v|to_add_out)|.*transformer_blocks\.[0-9]+\.attn\.to_out\.0|.*single_transformer_blocks\.[0-9]+\.attn\.to_out|.*single_transformer_blocks\.[0-9]+\.(proj_mlp|proj_out)|.*(?<!single_)transformer_blocks\.[0-9]+\.ff\.net\.2|.*(?<!single_)transformer_blocks\.[0-9]+\.ff\.net\.0\.proj|.*(?<!single_)transformer_blocks\.[0-9]+\.norm1_context\.linear|.*(?<!single_)transformer_blocks\.[0-9]+\.ff_context\.net\.0\.proj|.*(?<!single_)transformer_blocks\.[0-9]+\.ff_context\.net\.2|.*(?<!single_)transformer_blocks\.[0-9]+\.attn\.(to_add_out|add_k_proj|add_q_proj|add_v_proj))")


def _flux_pair(r, targets, guidance=True):
    from qflux_b200.flux_model import FluxB200, FluxB200Config
    kw = dict(num_layers=2, num_single_layers=2, attention_head_dim=128, num_attention_heads=2, joint_attention_dim=64,
              pooled_projection_dim=64, guidance_embeds=guidance)
    orc = mo.init_synthetic_(mo.FluxOracle(mo.FluxConfig(**kw)), std=0.05)
    g = torch.Generator().manual_seed(98)
    with torch.no_grad():
        for n, p in orc.named_parameters():
            if n.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.02)
            elif p.ndim == 1:
                p.copy_(1 + torch.randn(p.shape, generator=g) * 0.1)
    if r:
        mo.add_lora_adapter(orc, r=r, alpha=r, target_modules=targets, b_std=0.05)
    with torch.no_grad():
        for p in orc.parameters():
            p.copy_(p.bfloat16().float())
    m = FluxB200(FluxB200Config(**kw), device="cpu", _host_only=True)
    if r:
        m.add_adapter(r, r, target_modules=targets)
    missing, unexpected = m.load_state_dict(orc.state_dict(), strict=True)
    assert not missing and not unexpected, (missing, unexpected)
    assert set(m.state_dict()) == set(orc.state_dict())
    return orc, m


@pytest.mark.parametrize("targets", [("to_q", "to_k", "to_v", "to_out.0"),
                                     r".*(attn\.(to_[qkv]|add_[qkv]_proj|to_add_out)|proj_mlp|ff\.net\.0\.proj)",
                                     r".*(single_transformer_blocks\.[0-9]+\.(proj_mlp|proj_out)|ff\.net\.2|ff_context\.net\.(0\.proj|2)|attn\.to_out\.0)",
                                     FLUX_YAML_TARGETS])
def test_flux_step_matches_oracle_on_cpu(emu, targets):
    """BASELINE config 3 family (FLUX-Kontext shared-resolution recipe) at tiny size: 2 double + 2 single blocks."""
    from qflux_b200.train_step import FluxKontextStep
    orc, m = _flux_pair(4, targets)
    g = torch.Generator().manual_seed(3)
    rn = lambda *s: torch.randn(*s, generator=g).bfloat16()
    B, hw, T = 2, 4, 8
    L = hw * hw
    emb = dict(image_latents=rn(B, L, 64), control_latents=rn(B, L, 64), pooled_prompt_embeds=rn(B, 64), prompt_embeds=rn(B, T, 64),
               text_ids=torch.zeros(T, 3), image_ids=FluxKontextStep.latent_image_ids(hw, hw, "cpu", 0.0),
               control_ids=FluxKontextStep.latent_image_ids(hw, hw, "cpu", 1.0))
    noise, t = rn(B, L, 64), torch.tensor([0.5, 0.25])
    loss_o, pred_o = mo.flux_compute_loss_shared(orc, emb["image_latents"].float(), emb["control_latents"].float(),
                                                 emb["pooled_prompt_embeds"].float(), emb["prompt_embeds"].float(), emb["text_ids"],
                                                 emb["image_ids"], emb["control_ids"], noise=noise.float(), t=t)
    loss_o.backward()
    step = FluxKontextStep(m)
    loss_b = step.compute_loss(emb, noise=noise, t=t)
    pred_b = m._ws["pred"].view(B, -1, 64)[:, :L].float().clone()
    loss_b.backward()
    assert ((pred_b - pred_o).norm() / pred_o.norm()).item() < 1e-2
    assert abs(loss_b.item() - loss_o.item()) < 1e-2
    go = {n: (p.grad if p.grad is not None else torch.zeros_like(p)) for n, p in orc.named_parameters() if p.requires_grad}
    gb = {n: p.grad.float() for n, p in m.named_parameters()}
    assert set(go) == set(gb)
    num = sum(((gb[n] - go[n]) ** 2).sum() for n in go)
    den = sum((go[n] ** 2).sum() for n in go)
    assert float((num / den).sqrt()) < 2e-2


def test_flux_rope_table_matches_oracle():
    from qflux_b200.rope import flux_rope_table
    ids = torch.tensor([[0., 0, 0], [0, 1, 2], [1, 3, 0], [0, 0, 5]])
    cos, sin = mo.flux_rope(ids, (16, 56, 56))
    tab = flux_rope_table(ids)
    assert torch.equal(tab[..., 0], cos[:, 0::2]) and torch.equal(tab[..., 1], sin[:, 0::2])


def test_qwen_edit_plus_three_images_cumulative_rope(emu):
    """BASELINE config 4 semantics (Qwen-Image-Edit-2509 'Plus'): target + 2 control images, frame-axis RoPE offsets 0,1,2
    (transformer_qwenimage.py:213-224).  The trainer's `_compute_loss` is inherited unchanged (qwen_image_edit_plus_trainer.py)."""
    from qflux_b200.train_step import QwenImageEditStep
    orc, m = _pair(2, 2, 128, 4, ("to_q", "to_k", "to_v", "to_out.0"))
    g = torch.Generator().manual_seed(5)
    rn = lambda *s: torch.randn(*s, generator=g).bfloat16()
    B, T = 1, 16
    shapes = [[(1, 4, 4), (1, 4, 6), (1, 2, 4)]] * B  # target 16 tokens, controls 24 + 8 tokens of different sizes
    x = dict(image_latents=rn(B, 16, 64), control_latents=rn(B, 32, 64), prompt_embeds=rn(B, T, 128) * 3,
             prompt_embeds_mask=torch.ones(B, T, dtype=torch.int64), img_shapes=shapes, noise=rn(B, 16, 64), u=torch.tensor([0.25]))
    xf = {k: (v.float() if torch.is_tensor(v) and v.is_floating_point() and k != "u" else v) for k, v in x.items()}
    loss_o, pred_o = mo.qwen_compute_loss(orc, **xf)
    loss_o.backward()
    step = QwenImageEditStep(m)
    emb = {k: x[k] for k in ("image_latents", "control_latents", "prompt_embeds", "img_shapes")}
    loss_b = step.compute_loss(emb, noise=x["noise"], u=x["u"])
    pred_b = m._ws["pred"].view(B, -1, 64)[:, :16].float().clone()
    loss_b.backward()
    assert ((pred_b - pred_o).norm() / pred_o.norm()).item() < 1e-2
    go = {n: p.grad for n, p in orc.named_parameters() if p.requires_grad}
    num = sum(((p.grad.float() - go[n]) ** 2).sum() for n, p in m.named_parameters())
    den = sum((v ** 2).sum() for v in go.values())
    assert float((num / den).sqrt()) < 2e-2


def test_qwen_multi_resolution_matches_per_sample_oracle(emu):
    """BASELINE config 5 semantics (pad-to-max multi-resolution batch with per-sample RoPE, key masks for image AND text padding,
    AttentionMaskMseLoss over valid target tokens; transformer_qwen_custom.py:444-553, attention_mask_loss.py:146-226):
    the padded batch must equal the un-padded single-sample oracle runs (the reference's own self-check,
    tests/src/models/test_qwen_per_sample_rope.py:417)."""
    from qflux_b200.train_step import QwenImageEditStep
    orc, m = _pair(2, 2, 128, 4, ("to_q", "to_k", "to_v", "to_out.0"))
    g = torch.Generator().manual_seed(11)
    rn = lambda *s: torch.randn(*s, generator=g).bfloat16()
    shapes = [[(1, 4, 4), (1, 4, 4)], [(1, 2, 4), (1, 2, 4)]]
    lt, lc, T, txt = [16, 8], [16, 8], 8, [8, 5]
    x0, ctrl, pe, noise = rn(2, 16, 64), rn(2, 16, 64), rn(2, T, 128) * 3, rn(2, 16, 64)
    for t_ in (x0, ctrl, noise):
        t_[1, 8:] = 0
    pe[1, 5:] = 0
    mask = torch.tensor([[1] * 8, [1] * 5 + [0] * 3])
    u = torch.tensor([0.5, 0.25])
    sig = (1000 - (u * 1000).long()).float() / 1000
    # ---- oracle: one un-padded run per sample, AttentionMask-style normalisation over all valid target tokens
    preds, total = [], 0.0
    for b in range(2):
        s = sig[b]
        noisy = (1 - s) * x0[b, :lt[b]].float() + s * noise[b, :lt[b]].float()
        packed = torch.cat([noisy, ctrl[b, :lc[b]].float()], 0)[None]
        p = orc(hidden_states=packed, timestep=sig[b:b + 1], encoder_hidden_states=pe[b:b + 1, :txt[b]].float(),
                encoder_hidden_states_mask=mask[b:b + 1, :txt[b]], img_shapes=[shapes[b]], txt_seq_lens=[txt[b]])[0][0, :lt[b]]
        preds.append(p)
        total = total + ((p - (noise[b, :lt[b]].float() - x0[b, :lt[b]].float())) ** 2).mean(-1).sum()
    loss_o = total / (sum(lt) + 1e-12)
    loss_o.backward()
    # ---- fused model (emulated kernels): one padded batch
    step = QwenImageEditStep(m, "attention_mask")
    emb = dict(image_latents=x0, control_latents=ctrl, prompt_embeds=pe, prompt_embeds_mask=mask, img_shapes=shapes)
    loss_b = step.compute_loss(emb, noise=noise, u=u)
    pred_b = m._ws["pred"].view(2, -1, 64).float().clone()
    loss_b.backward()
    for b in range(2):
        assert ((pred_b[b, :lt[b]] - preds[b]).norm() / preds[b].norm()).item() < 1e-2
    assert abs(loss_b.item() - loss_o.item()) < 1e-2
    go = {n: p.grad for n, p in orc.named_parameters() if p.requires_grad}
    num = sum(((p.grad.float() - go[n]) ** 2).sum() for n, p in m.named_parameters())
    den = sum((v ** 2).sum() for v in go.values())
    assert float((num / den).sqrt()) < 2e-2
    # module API: padded output rows are exact zeros (tests/src/models/test_qwen_custom.py:672-692)
    packed = torch.zeros(2, 32, 64, dtype=torch.bfloat16)
    packed[0], packed[1, :16] = rn(32, 64), rn(16, 64)
    with torch.no_grad():
        out = m(hidden_states=packed, timestep=sig, encoder_hidden_states=pe, encoder_hidden_states_mask=mask, img_shapes=shapes,
                txt_seq_lens=txt)[0]
    assert out.shape == (2, 32, 64) and out[1, 16:].abs().max() == 0 and out[1, :16].abs().max() > 0
    # ... and the whole padded batch equals the oracle's restatement of the custom forward (transformer_qwen_custom.py:384-573)
    am = torch.zeros(2, 8 + 32, dtype=torch.bool)
    am[0], am[1, :5], am[1, 8:8 + 16] = True, True, True
    with torch.no_grad():
        ref = orc(hidden_states=packed.float(), timestep=sig, encoder_hidden_states=pe.float(), img_shapes=shapes, txt_seq_lens=txt,
                  attention_mask=am)[0]
    assert ((out.float() - ref).norm() / ref.norm()).item() < 1e-2 and ref[1, 16:].abs().max() == 0
    # the reference's own RoPE placement with padded text (transformer_qwen_custom.py:199-208: image table laid down right after the
    # un-padded text length) is available behind a switch and differs from the aligned placement exactly when text is padded
    with torch.no_grad():
        ref_r = orc(hidden_states=packed.float(), timestep=sig, encoder_hidden_states=pe.float(), img_shapes=shapes, txt_seq_lens=txt,
                    attention_mask=am, img_offset="reference")[0]
        m.rope_placement = "reference"
        out_r = m(hidden_states=packed, timestep=sig, encoder_hidden_states=pe, encoder_hidden_states_mask=mask, img_shapes=shapes,
                  txt_seq_lens=txt)[0]
        with pytest.raises(ValueError, match="txt_seq_lens"):
            m(hidden_states=packed, timestep=sig, encoder_hidden_states=pe, encoder_hidden_states_mask=mask, img_shapes=shapes)
        m.rope_placement = "aligned"
    assert ((out_r.float() - ref_r).norm() / ref_r.norm()).item() < 1e-2
    assert ((ref_r[1] - ref[1]).norm() / ref[1].norm()).item() > 2e-2, "sample 1 has padded text: the two placements must differ there"
    assert ((out_r[0].float() - out[0].float()).norm() / out[0].float().norm()).item() < 1e-2, "sample 0 has no text padding: same result"


def test_flux_multi_resolution_matches_per_sample_oracle(emu):
    """FLUX-Kontext pad-to-max multi-resolution recipe (flux_kontext_trainer.py:579-796, transformer_flux_custom.py): samples of
    different latent sizes in one padded batch with per-sample ids / RoPE, a key mask and a masked loss must equal running
    every sample alone and un-padded (the reference's own check: tests/src/models/test_flux_per_sample_rope.py:481-486)."""
    from qflux_b200.train_step import FluxKontextStep
    orc, m = _flux_pair(4, ("to_q", "to_k", "to_v", "to_out.0", "proj_mlp"))
    g = torch.Generator().manual_seed(21)
    rn = lambda *s: torch.randn(*s, generator=g).bfloat16()
    shapes = [[(1, 4, 4), (1, 4, 4)], [(1, 2, 4), (1, 4, 2)], [(1, 4, 2), (1, 2, 2), (1, 2, 4)]]
    B, T = 3, 8
    lt = [sh[0][1] * sh[0][2] for sh in shapes]
    lc = [sum(h * w for (_, h, w) in sh[1:]) for sh in shapes]
    Lm, Lcm = max(lt), max(lc)
    x0, ctrl, noise = rn(B, Lm, 64), rn(B, Lcm, 64), rn(B, Lm, 64)
    for b in range(B):
        x0[b, lt[b]:] = 0
        noise[b, lt[b]:] = 0
        ctrl[b, lc[b]:] = 0
    pe, pooled, t = rn(B, T, 64), rn(B, 64), torch.tensor([0.5, 0.25, 0.125])  # t * 1000 exact in bf16 (the model multiplies in bf16)
    text_ids = torch.zeros(T, 3)
    # ---- oracle: one un-padded run per sample; AttentionMaskMseLoss normalisation over all valid target tokens
    preds, total = [], 0.0
    for b in range(B):
        ids = [FluxKontextStep.latent_image_ids(shapes[b][0][1], shapes[b][0][2], "cpu", 0.0)]
        ids += [FluxKontextStep.latent_image_ids(h, w, "cpu", float(j + 1)) for j, (_, h, w) in enumerate(shapes[b][1:])]
        noisy = (1 - t[b]) * x0[b, :lt[b]].float() + t[b] * noise[b, :lt[b]].float()
        packed = torch.cat([noisy.bfloat16().float(), ctrl[b, :lc[b]].float()], 0)[None]
        p = orc(hidden_states=packed, encoder_hidden_states=pe[b:b + 1].float(), pooled_projections=pooled[b:b + 1].float(),
                timestep=t[b:b + 1], img_ids=torch.cat(ids, 0), txt_ids=text_ids, guidance=torch.ones(1))[0][0, :lt[b]]
        preds.append(p)
        total = total + ((p - (noise[b, :lt[b]].float() - x0[b, :lt[b]].float())) ** 2).mean(-1).sum()
    loss_o = total / (sum(lt) + 1e-12)
    loss_o.backward()
    # ---- fused model (emulated kernels): one padded batch
    step = FluxKontextStep(m, "attention_mask")
    emb = dict(image_latents=x0, control_latents=ctrl, pooled_prompt_embeds=pooled, prompt_embeds=pe, text_ids=text_ids, img_shapes=shapes)
    loss_b = step.compute_loss(emb, noise=noise, t=t)
    Ltot = max(a + c for a, c in zip(lt, lc))
    pred_b = m._ws["pred"].view(B, Ltot, 64).float().clone()
    loss_b.backward()
    for b in range(B):
        assert ((pred_b[b, :lt[b]] - preds[b]).norm() / preds[b].norm()).item() < 1e-2
    assert abs(loss_b.item() - loss_o.item()) < 1e-2
    go = {n: (p.grad if p.grad is not None else torch.zeros_like(p)) for n, p in orc.named_parameters() if p.requires_grad}
    num = sum(((p.grad.float() - go[n]) ** 2).sum() for n, p in m.named_parameters())
    den = sum((v ** 2).sum() for v in go.values())
    assert float((num / den).sqrt()) < 2e-2
    # "mse" criterion in this mode: mean over the padded [B, Lmax, C] block, padded elements contribute zero
    loss_m = FluxKontextStep(m, "mse").compute_loss(emb, noise=noise, t=t)
    assert abs(loss_m.item() - (total / (B * Lm)).item()) < 1e-2
    # module API (transformer_flux_custom.py signature): batched ids + attention_mask, padded rows come back as exact zeros
    ids_b = torch.zeros(B, Ltot, 3)
    am = torch.zeros(B, T + Ltot, dtype=torch.bool)
    for b in range(B):
        ids_b[b, :lt[b]] = FluxKontextStep.latent_image_ids(shapes[b][0][1], shapes[b][0][2], "cpu", 0.0)
        am[b, : T + lt[b] + lc[b]] = True
    hs_in = rn(B, Ltot, 64)
    with torch.no_grad():
        out = m(hidden_states=hs_in, encoder_hidden_states=pe, pooled_projections=pooled, timestep=t, img_ids=ids_b,
                txt_ids=text_ids, guidance=torch.ones(B), attention_mask=am)[0]
        # the oracle's restatement of the custom forward (transformer_flux_custom.py:372-741) on the same padded batch
        ref = orc(hidden_states=hs_in.float(), encoder_hidden_states=pe.float(), pooled_projections=pooled.float(), timestep=t, img_ids=ids_b,
                  txt_ids=text_ids, guidance=torch.ones(B), attention_mask=am)[0]
    assert out.shape == (B, Ltot, 64) and out[1, lt[1] + lc[1]:].abs().max() == 0 and out[1, : lt[1]].abs().max() > 0
    assert ((out.float() - ref).norm() / ref.norm()).item() < 1e-2 and ref[1, lt[1] + lc[1]:].abs().max() == 0


def test_fused_adamw_matches_torch_adamw(emu):
    """FusedLoraAdamW (clip + AdamW on the flat fp32 gradient; SURVEY.md §8 f1) against clip_grad_norm_ + torch.optim.AdamW run on
    fp32 master copies of the same parameters, three steps; bf16 parameters agree to one rounding."""
    from qflux_b200.optim import FusedLoraAdamW
    from qflux_b200.train_step import QwenImageEditStep
    orc, m = _pair(2, 2, 128, 4, ("to_q", "to_out.0", "img_mod.1", "net.2"))
    x = _inputs(2, 4, 24, 128)
    emb = {k: x[k] for k in ("image_latents", "control_latents", "prompt_embeds", "prompt_embeds_mask", "img_shapes")}
    step = QwenImageEditStep(m, "mse", max_grad_norm=0.05)  # small enough that clipping is active
    opt = FusedLoraAdamW(m, lr=1e-2, weight_decay=0.1)
    master = {n: p.detach().float().clone().requires_grad_(True) for n, p in m.named_parameters()}
    ref = torch.optim.AdamW(list(master.values()), lr=1e-2, weight_decay=0.1)
    for it in range(3):
        before = {n: p.detach().float().clone() for n, p in m.named_parameters()}
        step.train_step(emb, opt, noise=x["noise"], u=x["u"])
        gv = m.lora_grad_views()  # the fp32 accumulator the fused kernel consumed
        for n, p in master.items():
            p.data.copy_(before[n])  # same starting point as the bf16 parameters of this step
            p.grad = gv[n].clone()
        norm = torch.nn.utils.clip_grad_norm_(list(master.values()), 0.05)
        assert abs(float(opt.grad_norm_sq.sqrt()) - float(norm)) < 1e-4 * float(norm) and float(norm) > 0.05
        ref.step()
        for n, p in m.named_parameters():
            assert torch.equal(p.detach(), master[n].detach().to(torch.bfloat16)) or \
                (p.detach().float() - master[n].detach()).abs().max() <= 2 * 2 ** -8 * master[n].detach().abs().max(), n
    # it is a torch Optimizer: LR schedulers drive it, and its state round-trips
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda k: 0.5 ** k)
    step.train_step(emb, opt, noise=x["noise"], u=x["u"])
    sched.step()
    assert abs(opt.param_groups[0]["lr"] - 0.5e-2) < 1e-12 and opt.step_count == 4
    sd = opt.state_dict()
    assert set(sd) == {"state", "param_groups", "fused"} and sd["fused"]["step"] == 4
    opt2 = FusedLoraAdamW(m, lr=1.0)
    opt2.load_state_dict(sd)
    assert opt2.step_count == 4 and opt2.param_groups[0]["lr"] == opt.param_groups[0]["lr"] and torch.equal(opt2.exp_avg, opt.exp_avg)


def test_sampling_loops_match_oracle(emu):
    """Inference sampler (SURVEY.md §8 f2): the same Euler / true-CFG loop driven by the fused model (emulated kernels) and by the
    oracle must agree; schedule sanity: decreasing sigmas from the shifted 1.0 to 0, more shift for longer sequences."""
    from qflux_b200 import sampler
    sig = sampler.flow_match_sigmas(8, 1024)
    assert sig.shape == (9,) and sig[-1] == 0 and abs(float(sig[0]) - 1.0) < 1e-6 and bool((sig[1:] < sig[:-1]).all())
    assert float(sampler.flow_match_sigmas(8, 4096)[4]) > float(sig[4]) > float(sampler.flow_match_sigmas(8, 256)[4])
    assert abs(sampler.calculate_shift(256) - 0.5) < 1e-9 and abs(sampler.calculate_shift(4096) - 1.15) < 1e-9
    g = torch.Generator().manual_seed(5)
    rn = lambda *s: torch.randn(*s, generator=g).bfloat16()
    # ---- Qwen, true CFG with norm rescaling
    orc, m = _pair(2, 2, 128, 4, ("to_q", "to_k", "to_v", "to_out.0"))
    B, hw, T = 2, 4, 8
    emb = dict(latents=rn(B, hw * hw, 64), control_latents=rn(B, hw * hw, 64), prompt_embeds=rn(B, T, 128) * 3,
               prompt_embeds_mask=torch.ones(B, T, dtype=torch.int64), negative_prompt_embeds=rn(B, T, 128) * 3,
               negative_prompt_embeds_mask=torch.ones(B, T, dtype=torch.int64), img_shapes=[[(1, hw, hw), (1, hw, hw)]] * B,
               num_inference_steps=3, true_cfg_scale=2.5)

    class F32:  # the oracle behind the module signature, bf16 in / bf16 out like a bf16 model
        def __init__(self, net):
            self.net, self.device = net, torch.device("cpu")

        def __call__(self, **kw):
            if "pooled_projections" in kw:  # a bf16 FLUX model multiplies timestep / guidance by 1000 IN bf16 (transformer_flux.py:707-710)
                for k in ("timestep", "guidance"):
                    kw[k] = (kw[k].bfloat16() * 1000).float() / 1000
            kw = {k: (v.float() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in kw.items()}
            if "txt_seq_lens" in kw and kw["txt_seq_lens"] is None:
                kw["txt_seq_lens"] = kw["encoder_hidden_states_mask"].sum(1).tolist()
            with torch.no_grad():
                return (self.net(**kw)[0].bfloat16(),)

    out_b = sampler.sample_qwen(m, emb)
    out_o = sampler.sample_qwen(F32(orc), emb)
    assert out_b.shape == (B, hw * hw, 64) and ((out_b.float() - out_o.float()).norm() / out_o.float().norm()).item() < 2e-2
    # ---- FLUX
    from qflux_b200.train_step import FluxKontextStep
    forc, fm = _flux_pair(4, ("to_q", "to_k", "to_v", "to_out.0"))
    femb = dict(latents=rn(B, hw * hw, 64), latent_ids=FluxKontextStep.latent_image_ids(hw, hw, "cpu", 0.0),
                control_latents=rn(B, hw * hw, 64), control_ids=FluxKontextStep.latent_image_ids(hw, hw, "cpu", 1.0),
                pooled_prompt_embeds=rn(B, 64), prompt_embeds=rn(B, T, 64), text_ids=torch.zeros(T, 3), guidance=3.5,
                negative_pooled_prompt_embeds=rn(B, 64), negative_prompt_embeds=rn(B, T, 64), negative_text_ids=torch.zeros(T, 3),
                num_inference_steps=3, true_cfg_scale=1.5)
    fo_b = sampler.sample_flux(fm, femb)
    fo_o = sampler.sample_flux(F32(forc), femb)
    assert ((fo_b.float() - fo_o.float()).norm() / fo_o.float().norm()).item() < 2e-2


def test_gradient_accumulation_equals_one_big_batch(emu):
    """train.gradient_accumulation_steps (accelerator.accumulate, base_trainer.py:518-533): two micro-steps of B=1 accumulate into the same
    flat gradient and step once with the mean — the same update as one step on the B=2 batch (MSE: mean over samples)."""
    from qflux_b200.optim import FusedLoraAdamW
    from qflux_b200.train_step import QwenImageEditStep
    res = {}
    x = _inputs(2, 4, 24, 128)
    keys = ("image_latents", "control_latents", "prompt_embeds", "prompt_embeds_mask")
    for mode in ("big", "accum"):
        orc, m = _pair(2, 2, 128, 4, ("to_q", "to_out.0"))
        opt = FusedLoraAdamW(m, lr=1e-2, weight_decay=0.0)
        if mode == "big":
            step = QwenImageEditStep(m, "mse", max_grad_norm=0.0)
            step.train_step({**{k: x[k] for k in keys}, "img_shapes": x["img_shapes"]}, opt, noise=x["noise"], u=x["u"])
        else:
            step = QwenImageEditStep(m, "mse", max_grad_norm=0.0, gradient_accumulation_steps=2)
            p0 = [p.detach().clone() for p in m.parameters()]
            for b in range(2):
                emb = {**{k: x[k][b:b + 1] for k in keys}, "img_shapes": x["img_shapes"][b:b + 1]}
                step.train_step(emb, opt, noise=x["noise"][b:b + 1], u=x["u"][b:b + 1])
                if b == 0:  # no optimizer step after the first micro-step
                    assert all(torch.equal(p, q) for p, q in zip(m.parameters(), p0)) and opt.step_count == 0
            assert opt.step_count == 1
        res[mode] = (m.G32.clone(), [p.detach().float().clone() for p in m.parameters()])
    g_big, g_acc = res["big"][0], res["accum"][0] / 2  # the accumulator holds the SUM over micro-steps; the optimizer divides
    assert ((g_big - g_acc).norm() / g_big.norm()).item() < 2e-2
    num = sum(((a - b) ** 2).sum() for a, b in zip(res["big"][1], res["accum"][1]))
    den = sum((a ** 2).sum() for a in res["big"][1])
    assert float((num / den).sqrt()) < 1e-3


def test_backward_of_a_stale_forward_is_refused(emu):
    """One activation workspace per model: a second forward overwrites what the first forward's backward would read, so that backward
    raises instead of producing gradients from the wrong activations; train_step's loss is a private copy."""
    from qflux_b200.train_step import QwenImageEditStep
    orc, m = _pair(2, 1, 128, 4, ("to_q", "to_k", "to_v", "to_out.0"))
    x = _inputs(1, 4, 24, 128)
    packed = torch.cat([x["image_latents"], x["control_latents"]], 1)
    kw = dict(timestep=torch.tensor([0.625]), encoder_hidden_states_mask=x["prompt_embeds_mask"], img_shapes=x["img_shapes"], txt_seq_lens=[24],
              encoder_hidden_states=x["prompt_embeds"])
    p1 = m(hidden_states=packed, **kw)[0]
    p2 = m(hidden_states=packed * 0.5, **kw)[0]
    with pytest.raises(RuntimeError, match="overwritten by a later forward"):
        p1.float().pow(2).mean().backward()
    p2.float().pow(2).mean().backward()  # the most recent forward is fine
    step = QwenImageEditStep(m)
    emb = {k: x[k] for k in ("image_latents", "control_latents", "prompt_embeds", "img_shapes")}
    l1 = step.compute_loss(emb, noise=x["image_latents"], u=torch.tensor([0.5]))
    step.compute_loss(emb, noise=x["image_latents"], u=torch.tensor([0.25]))
    with pytest.raises(RuntimeError, match="overwritten by a later forward"):
        l1.backward()
    a = step.train_step(emb, noise=x["image_latents"], u=torch.tensor([0.5]))
    a0 = float(a)
    step.train_step(emb, noise=x["image_latents"], u=torch.tensor([0.25]))
    assert float(a) == a0, "train_step must return its own copy of the loss, not the workspace scalar"


def test_row_band_plan_properties():
    """lib.RowBands.plan (ragged GEMM rows of a pad-to-max batch): bands are disjoint 256-row spans, every valid row is inside a band, the
    dead ranges are exactly the complement inside [0, M), and nothing is planned when nothing can be skipped."""
    from hypothesis import given, settings, strategies as st
    from qflux_b200.lib import RowBands

    @settings(max_examples=300, deadline=None)
    @given(st.integers(1, 6).flatmap(lambda B: st.tuples(st.just(B), st.integers(1, 2000))).flatmap(
        lambda br: st.tuples(st.just(br[1]), st.lists(st.integers(0, br[1]), min_size=br[0], max_size=br[0]))))
    def check(rv):
        R, valid = rv
        M = R * len(valid)
        plan = RowBands.plan(valid, R)
        covered = [False] * M
        if plan is None:  # nothing to skip: the bands of the dense tiling would cover every row
            live = set()
            for b, v in enumerate(valid):
                live.update(range(b * R, b * R + v))
            # a plan is only omitted when there is no dead range, i.e. the 256-row bands over the merged valid intervals reach M
            assert M - len(live) < 256 * len(valid) + 256
            return
        tiles, dead = plan
        assert tiles == sorted(tiles) and all(b - a >= 256 for a, b in zip(tiles, tiles[1:])), "bands overlap"
        for t in tiles:
            for r in range(t, min(t + 256, M)):
                covered[r] = True
        for b, v in enumerate(valid):
            assert all(covered[b * R: b * R + v]), "a valid row is outside every band"
        dead_rows = set()
        for lo, hi in dead:
            assert 0 <= lo < hi <= M
            dead_rows.update(range(lo, hi))
        assert dead_rows == {r for r in range(M) if not covered[r]}, "dead ranges must be the complement of the bands"
        assert dead, "a plan without dead ranges should have been None"
    check()


def test_multi_resolution_row_bands_equal_pad_to_max(emu, monkeypatch):
    """Host-side plumbing of the ragged GEMM row bands (emulated kernels zero-fill the skipped rows like qfx_zero_rows): a pad-to-max batch
    whose padding spans whole 256-row bands must give the loss and LoRA gradients of the dense pad-to-max run — the padded rows carry
    exact zeros through every gradient buffer either way."""
    from qflux_b200.train_step import QwenImageEditStep
    g = torch.Generator().manual_seed(17)
    rn = lambda *s: torch.randn(*s, generator=g).bfloat16()
    shapes = [[(1, 24, 16), (1, 24, 16)], [(1, 8, 8), (1, 8, 8)], [(1, 16, 16), (1, 16, 16)]]
    lt = [sh[0][1] * sh[0][2] for sh in shapes]
    B, T, txt, Lt = 3, 8, [8, 5, 7], max(lt)
    x0, ctrl, pe, noise = rn(B, Lt, 64), rn(B, Lt, 64), rn(B, T, 128) * 3, rn(B, Lt, 64)
    mask = torch.zeros(B, T, dtype=torch.int64)
    for b in range(B):
        x0[b, lt[b]:] = 0; ctrl[b, lt[b]:] = 0; noise[b, lt[b]:] = 0; pe[b, txt[b]:] = 0; mask[b, :txt[b]] = 1
    emb = dict(image_latents=x0, control_latents=ctrl, prompt_embeds=pe, prompt_embeds_mask=mask, img_shapes=shapes)
    u = torch.tensor([0.5, 0.25, 0.75])
    out = {}
    for mode in ("bands", "dense"):
        if mode == "dense":
            monkeypatch.setenv("QFX_NO_RAGGED_GEMM", "1")
        orc, m = _pair(2, 2, 128, 4, ("to_q", "to_k", "to_v", "to_out.0", "img_mlp.net.2"))
        step = QwenImageEditStep(m, "attention_mask")
        loss = step.compute_loss(emb, noise=noise, u=u)
        loss.backward()
        bands = m._ws.get("bands")
        assert (bands is not None and bands.n_dead > 0) == (mode == "bands")
        out[mode] = (float(loss), m.G32.clone(), m._ws["pred"].float().clone())
    assert out["bands"][0] == out["dense"][0]
    assert ((out["bands"][1] - out["dense"][1]).norm() / out["dense"][1].norm()).item() < 1e-6
    valid = torch.zeros(B, Lt, dtype=torch.bool)
    for b in range(B):
        valid[b, :lt[b]] = True
    pb, pd = (o[2].view(B, 2 * Lt, 64)[:, :Lt][valid] for o in (out["bands"], out["dense"]))
    assert torch.equal(pb, pd)


def test_workspaces_are_kept_per_shape(emu):
    """One training workspace and up to three inference workspaces stay allocated: alternating prompt lengths (true CFG) or a validation
    pass between training steps must hand back the SAME buffers, because CUDA graphs captured on them hold raw pointers."""
    from qflux_b200.train_step import QwenImageEditStep
    orc, m = _pair(2, 1, 128, 4, ("to_q", "to_k", "to_v", "to_out.0"))
    x = _inputs(1, 4, 24, 128)
    packed = torch.cat([x["image_latents"], x["control_latents"]], 1)

    def infer(T):
        pe = x["prompt_embeds"][:, :T]
        with torch.no_grad():
            m(hidden_states=packed, timestep=torch.tensor([0.5]), encoder_hidden_states=pe, img_shapes=x["img_shapes"],
              encoder_hidden_states_mask=torch.ones(1, T, dtype=torch.int64))
        return m._ws
    a, b = infer(24), infer(17)
    assert a is not b and infer(24) is a and infer(17) is b and len(m._infer_ws) == 2
    step = QwenImageEditStep(m)
    emb = {k: x[k] for k in ("image_latents", "control_latents", "prompt_embeds", "img_shapes")}
    step.train_step(emb, noise=x["image_latents"], u=torch.tensor([0.5]))
    train_ws = m._ws
    assert m._train_ws[1] is train_ws and train_ws is not a
    assert infer(24) is a                     # validation in between ...
    step.train_step(emb, noise=x["image_latents"], u=torch.tensor([0.5]))
    assert m._ws is train_ws                  # ... and training resumes on the buffers it had
    for T in (9, 10, 11):                     # a fourth inference shape evicts the oldest one only
        infer(T)
    assert len(m._infer_ws) == 3 and m._activate_ws(train_ws, m._train_ws[0]) and not m._activate_ws(a, (1, 24, 32, False))
