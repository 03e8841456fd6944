"""GPU parity of the fused Qwen-Image training step against the pure-torch oracle (run under gpurun).

The oracle runs on the same GPU in fp32 (reference numerics) and in bf16 (the reference's eager working dtype); the
fused path is compared with both using the reference's own metric, relative L2 (tests/src/models/test_qwen_custom.py:550).
"""
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from harness import main, rel_l2  # noqa: E402
from lora_grad_check import eager_sdpa, per_tensor  # noqa: E402

import torch  # noqa: E402


def build_pair(H, L, J, r, targets, seed=0, b_std=0.05, w_std=0.05):
    from oracle import mmdit_oracle as mo
    from qflux_b200.qwen_model import QwenB200Config, QwenImageB200
    cfg = mo.QwenConfig(num_layers=L, attention_head_dim=128, num_attention_heads=H, joint_attention_dim=J)
    orc = mo.init_synthetic_(mo.QwenImageOracle(cfg), seed=1234 + seed, std=w_std)
    # make norm weights / biases non-trivial so the parity test exercises them
    g = torch.Generator().manual_seed(99)
    with torch.no_grad():
        for n, p in orc.named_parameters():
            if n.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.02)
            elif p.ndim == 1:
                p.copy_(1 + torch.randn(p.shape, generator=g) * 0.1)
    if r:
        mo.add_lora_adapter(orc, r=r, alpha=r, target_modules=targets, seed=seed, b_std=b_std)
    orc = orc.cuda()
    # quantise every parameter to bf16 once so that fp32-oracle, bf16-oracle and the fused model share identical weights
    with torch.no_grad():
        for p in orc.parameters():
            p.copy_(p.bfloat16().float())
    m = QwenImageB200(QwenB200Config(num_layers=L, num_attention_heads=H, joint_attention_dim=J))
    if r:
        m.add_adapter(r, r, target_modules=targets)
    missing, unexpected = m.load_state_dict(orc.state_dict(), strict=True)
    assert not unexpected and not missing, (missing, unexpected)
    return orc, m


def inputs(B, hw, T, J, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    L = hw * hw
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g).bfloat16()
    return dict(image_latents=rn(B, L, 64), control_latents=rn(B, L, 64), prompt_embeds=rn(B, T, J) * 3,
                prompt_embeds_mask=torch.ones(B, T, dtype=torch.int64, device="cuda"),
                img_shapes=[[(1, hw, hw), (1, hw, hw)]] * B, noise=rn(B, L, 64),
                u=torch.tensor([0.5, 0.25, 0.125, 0.75][:B]))  # sigma .5/.75/.875/.25: exact in bf16


def _grad_per_tensor(res, gb, g_o, g_h):
    """Each LoRA gradient tensor of the fused step against the fp32 oracle, scaled by the bf16 oracle's own error for that tensor
    (lora_grad_check.per_tensor): a pooled norm over all tensors would hide a wrong small one."""
    pt = per_tensor(gb, g_o, g_h)
    res["grad_tensor_fail"], res["grad_worst_ratio"] = pt["fail"], pt["worst_ratio"]


def step_parity(H=2, L=2, J=128, B=2, hw=4, T=24, r=4, targets=("to_q", "to_k", "to_v", "to_out.0"), bf16_oracle=True):
    from oracle import mmdit_oracle as mo
    from qflux_b200.train_step import QwenImageEditStep
    orc, m = build_pair(H, L, J, r, targets)
    x = inputs(B, hw, T, J)
    res = {}
    # ---- fp32 oracle
    xf = {k: (v.float() if torch.is_tensor(v) and v.is_floating_point() and k != "u" else v) for k, v in x.items()}
    loss_o, pred_o = mo.qwen_compute_loss(orc, **xf)
    loss_o.backward()
    g_o = {n: (p.grad.clone() if p.grad is not None else torch.zeros_like(p)) for n, p in orc.named_parameters() if p.requires_grad}
    # ---- fused model
    step = QwenImageEditStep(m)
    emb = {k: x[k] for k in ("image_latents", "control_latents", "prompt_embeds", "img_shapes")}
    loss_b = step.compute_loss(emb, noise=x["noise"], u=x["u"])
    pred_b = m._ws["pred"].view(B, -1, 64)[:, : hw * hw].float().clone()
    loss_b.backward()
    torch.cuda.synchronize()
    res["pred_vs_fp32"] = rel_l2(pred_b, pred_o)
    res["loss_abs"] = abs(loss_b.item() - loss_o.item())
    res["loss"] = loss_o.item()
    res["loss_rel"] = res["loss_abs"] / max(1.0, abs(loss_o.item()))
    gb = {n: p.grad.float() for n, p in m.named_parameters()}
    assert set(gb) == set(g_o), (set(gb) ^ set(g_o))
    num = sum(((gb[n] - g_o[n]).double() ** 2).sum() for n in g_o)
    den = sum((g_o[n].double() ** 2).sum() for n in g_o)
    res["grad_vs_fp32"] = float((num / den).sqrt())
    res["grad_worst"] = max(rel_l2(gb[n], g_o[n]) for n in g_o if g_o[n].abs().max() > 0)
    # fast path must give the same gradients as the autograd path
    step.train_step(emb, noise=x["noise"], u=x["u"])
    gv = m.lora_grad_views()
    res["fast_vs_autograd"] = max(rel_l2(gv[n], gb[n]) for n in gb if gb[n].abs().max() > 0)
    # ---- bf16 oracle (what the reference actually runs on a GPU)
    if bf16_oracle:
        orc.zero_grad()
        orc16 = orc.bfloat16()
        with eager_sdpa():
            loss_h, pred_h = mo.qwen_compute_loss(orc16, **x)
            loss_h.backward()
        g_h = {n: (p.grad.float() if p.grad is not None else torch.zeros_like(p).float()) for n, p in orc16.named_parameters() if p.requires_grad}
        res["bf16oracle_pred_vs_fp32"] = rel_l2(pred_h.float(), pred_o)
        res["pred_vs_bf16oracle"] = rel_l2(pred_b, pred_h.float())
        num = sum(((g_h[n] - g_o[n]).double() ** 2).sum() for n in g_o)
        res["bf16oracle_grad_vs_fp32"] = float((num / den).sqrt())
        _grad_per_tensor(res, gb, g_o, g_h)
    res["err"] = max(res["pred_vs_fp32"], res["grad_vs_fp32"])
    return res


def inference_parity():
    """no-grad forward through the public module signature (the `dit(...)` call of the trainer)."""
    orc, m = build_pair(2, 2, 128, 0, None)
    x = inputs(2, 4, 24, 128)
    packed = torch.cat([x["image_latents"], x["control_latents"]], 1)
    t = torch.tensor([0.75, 0.25], device="cuda")
    with torch.no_grad():
        po = orc(hidden_states=packed.float(), timestep=t, encoder_hidden_states=x["prompt_embeds"].float(),
                 encoder_hidden_states_mask=x["prompt_embeds_mask"], img_shapes=x["img_shapes"], txt_seq_lens=[24, 24])[0]
        pb = m(hidden_states=packed, timestep=t, guidance=None, encoder_hidden_states_mask=x["prompt_embeds_mask"],
               encoder_hidden_states=x["prompt_embeds"], img_shapes=x["img_shapes"], txt_seq_lens=[24, 24], return_dict=False)[0]
    return dict(err=rel_l2(pb.float(), po))


def full_width_block():
    """One full-width Qwen block (D=3072, H=24) at the benchmark sequence shape, B=1."""
    t0 = time.time()
    r = step_parity(H=24, L=1, J=3584, B=1, hw=32, T=352, r=16, bf16_oracle=True)
    r["secs"] = round(time.time() - t0, 1)
    return r


def bench_point_6blk():
    """The benchmark point (SURVEY.md §8d cfg 2) at reduced DEPTH only: 6 full-width Qwen blocks (D=3072, H=24), B=4, T=352, 2 x 1024
    image tokens, LoRA r=16 — fused step vs the fp32 and the bf16 oracle (cross-block strides, the B=4 batch indexing of the modulation
    vectors, the grouped text+image launches at their real sizes).  Also the ragged-mask variant [352, 300, 352, 257]: the stock Qwen
    forward hands `attention_mask=None` to SDPA and uses only max(txt_seq_lens) for the RoPE table (transformer_qwenimage.py:226-232,
    332-339), so its result must EQUAL the all-ones-mask result — checked on the oracle and on the fused module path."""
    from oracle import mmdit_oracle as mo
    t0 = time.time()
    r = step_parity(H=24, L=6, J=3584, B=4, hw=32, T=352, r=16, bf16_oracle=True)
    torch.cuda.empty_cache()
    # ragged text mask through the public module signature (2 blocks are enough: the mask never reaches a kernel in this mode)
    orc, m = build_pair(24, 2, 3584, 0, None)
    x = inputs(4, 32, 352, 3584)
    packed = torch.cat([x["image_latents"], x["control_latents"]], 1)
    t = torch.tensor([0.75, 0.25, 0.5, 0.125], device="cuda")
    ragged = torch.zeros(4, 352, dtype=torch.int64, device="cuda")
    for b, n in enumerate([352, 300, 352, 257]):
        ragged[b, :n] = 1
    with torch.no_grad():
        outs = {}
        for name, mask in (("ones", x["prompt_embeds_mask"]), ("ragged", ragged)):
            lens = mask.sum(1).tolist()
            outs["orc_" + name] = orc.bfloat16()(hidden_states=packed, timestep=t, encoder_hidden_states=x["prompt_embeds"],
                                                  encoder_hidden_states_mask=mask, img_shapes=x["img_shapes"], txt_seq_lens=lens)[0].float()
            outs["b200_" + name] = m(hidden_states=packed, timestep=t, guidance=None, encoder_hidden_states_mask=mask,
                                     encoder_hidden_states=x["prompt_embeds"], img_shapes=x["img_shapes"], txt_seq_lens=lens,
                                     return_dict=False)[0].float()
    r["ragged_mask_oracle_diff"] = float((outs["orc_ragged"] - outs["orc_ones"]).abs().max())
    # (the split-K tail of the GEMMs adds partial sums with red.global in arrival order: two launches differ in the last bf16 bit here and
    # there, so the fused comparison is a relative L2 against that run-to-run floor, not bit equality)
    r["ragged_mask_b200_diff"] = rel_l2(outs["b200_ragged"], outs["b200_ones"])
    r["ragged_b200_vs_bf16oracle"] = rel_l2(outs["b200_ragged"], outs["orc_ragged"])
    r["secs"] = round(time.time() - t0, 1)
    return r


def train_trajectory(steps=5, H=4, L=4, J=256, B=4, hw=8, T=40, r=8):
    """`steps` optimizer steps: fused step + FusedLoraAdamW (clip 1.0) on the fused path vs the fp32 oracle + clip_grad_norm_ +
    torch.optim.AdamW with the same noise / timestep draws — loss trajectory and final LoRA parameters."""
    from oracle import mmdit_oracle as mo
    from qflux_b200.optim import FusedLoraAdamW
    from qflux_b200.train_step import QwenImageEditStep
    orc, m = build_pair(H, L, J, r, ("to_q", "to_k", "to_v", "to_out.0"))
    x = inputs(B, hw, T, J)
    xf = {k: (v.float() if torch.is_tensor(v) and v.is_floating_point() and k != "u" else v) for k, v in x.items()}
    emb = {k: x[k] for k in ("image_latents", "control_latents", "prompt_embeds", "img_shapes")}
    lr, wd = 2e-3, 1e-2
    params = [p for p in orc.parameters() if p.requires_grad]
    ref_opt = torch.optim.AdamW(params, lr=lr, weight_decay=wd)
    step, opt = QwenImageEditStep(m, max_grad_norm=1.0), FusedLoraAdamW(m, lr=lr, weight_decay=wd)
    g = torch.Generator(device="cuda").manual_seed(7)
    us = [torch.tensor([0.5, 0.25, 0.125, 0.75]), torch.tensor([0.75, 0.5, 0.25, 0.125]), torch.tensor([0.125, 0.75, 0.5, 0.25])]
    lo, lb = [], []
    for it in range(steps):
        noise = torch.randn(B, hw * hw, 64, device="cuda", generator=g).bfloat16()
        u = us[it % 3][:B]
        loss_o, _ = mo.qwen_compute_loss(orc, **{**xf, "noise": noise.float(), "u": u})
        ref_opt.zero_grad()
        loss_o.backward()
        torch.nn.utils.clip_grad_norm_(params, 1.0)
        ref_opt.step()
        lo.append(loss_o.item())
        lb.append(float(step.train_step(emb, opt, noise=noise, u=u).item()))
    torch.cuda.synchronize()
    po = {n: p.detach() for n, p in orc.named_parameters() if p.requires_grad}
    num = sum(((p.detach().float() - po[n]).double() ** 2).sum() for n, p in m.named_parameters())
    den = sum((v.double() ** 2).sum() for v in po.values())
    return dict(loss_oracle=lo, loss_b200=lb, loss_max_rel=max(abs(a - b) / max(1.0, abs(a)) for a, b in zip(lo, lb)),
                param_rel=float((num / den).sqrt()), decreased=lb[-1] < lb[0], err=max(abs(a - b) / max(1.0, abs(a)) for a, b in zip(lo, lb)))


def graph_replay():
    """The CUDA-graph-captured step (second and later calls of `train_step`) must reproduce the eager step: same loss and LoRA gradients
    for the same inputs (the attention backward accumulates dQ with atomics, so 'same' is to a few fp32 ulps of reordering), new inputs
    must be picked up through the static buffers, and the launch counter must keep counting.  Qwen and FLUX (YAML target set: the path
    with AdaLN-linear LoRA, whose index bookkeeping must stay off the host inside the capture)."""
    from qflux_b200 import lib
    from qflux_b200.train_step import FluxKontextStep, QwenImageEditStep
    res = {}
    orc, m = build_pair(2, 2, 128, 4, ("to_q", "to_k", "to_v", "to_out.0", "img_mod.1"))
    x = inputs(2, 4, 24, 128)
    emb = {k: x[k] for k in ("image_latents", "control_latents", "prompt_embeds", "img_shapes")}
    eager, graphed = QwenImageEditStep(m, use_cuda_graph=False), QwenImageEditStep(m, use_cuda_graph=True)
    l_e = float(eager.train_step(emb, noise=x["noise"], u=x["u"]))
    g_e = m.G32.clone()
    n0 = lib.LAUNCHES
    l1 = float(graphed.train_step(emb, noise=x["noise"], u=x["u"]))   # eager warm-up of the graphed step object
    per_step = lib.LAUNCHES - n0
    l2 = float(graphed.train_step(emb, noise=x["noise"], u=x["u"]))   # capture + first replay
    g2 = m.G32.clone()
    l3 = float(graphed.train_step(emb, noise=x["noise"], u=x["u"]))   # replay
    res["qwen_loss"] = max(abs(l_e - l1), abs(l_e - l2), abs(l_e - l3))
    res["qwen_grad"] = max(rel_l2(g2, g_e), rel_l2(m.G32, g_e))
    res["launch_count_ok"] = float(lib.LAUNCHES - n0 != 3 * per_step)
    noise2 = (x["noise"].float() * 0.5).bfloat16()
    l_new_e = float(eager.train_step(emb, noise=noise2, u=x["u"]))
    g_new_e = m.G32.clone()
    l_new_g = float(graphed.train_step(emb, noise=noise2, u=x["u"]))
    res["qwen_new_inputs"] = max(abs(l_new_e - l_new_g), rel_l2(m.G32, g_new_e))
    assert abs(l_new_e - l_e) > 1e-3, "the second input set must actually differ"
    assert len(graphed._graphs.entries) == 1 and graphed._graphs.captured() == 1, "no graph was captured"
    # FLUX with the YAML target regex
    orc, mf = build_flux_pair(targets=FLUX_YAML_TARGETS, r=4)
    g = torch.Generator(device="cuda").manual_seed(3)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g).bfloat16()
    B, hw, T = 2, 4, 8
    embf = dict(image_latents=rn(B, hw * hw, 64), control_latents=rn(B, hw * hw, 64), pooled_prompt_embeds=rn(B, 64), prompt_embeds=rn(B, T, 64),
                text_ids=torch.zeros(T, 3, device="cuda"), image_ids=FluxKontextStep.latent_image_ids(hw, hw, "cuda", 0.0),
                control_ids=FluxKontextStep.latent_image_ids(hw, hw, "cuda", 1.0))
    nz, t = rn(B, hw * hw, 64), torch.tensor([0.5, 0.25], device="cuda")
    fe, fg = FluxKontextStep(mf, use_cuda_graph=False), FluxKontextStep(mf, use_cuda_graph=True)
    le = float(fe.train_step(embf, noise=nz, t=t))
    ge = mf.G32.clone()
    ls = [float(fg.train_step(embf, noise=nz, t=t)) for _ in range(3)]
    res["flux_loss"] = max(abs(le - v) for v in ls)
    res["flux_grad"] = rel_l2(mf.G32, ge)
    assert len(fg._graphs.entries) == 1 and fg._graphs.captured() == 1, "no FLUX graph was captured"
    res["err"] = max(res.values())
    return res


def grad_accum():
    """`gradient_accumulation_steps=2` on the CUDA path (graphs on: the accumulating and the non-accumulating micro-step are two different
    captured graphs): two B=1 micro-steps must give the gradient and the parameter update of one B=2 step (accelerator.accumulate
    semantics, base_trainer.py:518-533), repeated so that the replays are exercised too."""
    from qflux_b200.optim import FusedLoraAdamW
    from qflux_b200.train_step import QwenImageEditStep
    keys = ("image_latents", "control_latents", "prompt_embeds")
    x = inputs(2, 8, 24, 128)
    out = {}
    for mode in ("big", "accum"):
        orc, m = build_pair(2, 2, 128, 4, ("to_q", "to_k", "to_v", "to_out.0"))
        opt = FusedLoraAdamW(m, lr=1e-2, weight_decay=0.0)
        gs = []
        if mode == "big":
            step = QwenImageEditStep(m, "mse", max_grad_norm=0.0)
            for it in range(3):
                step.train_step({**{k: x[k] for k in keys}, "img_shapes": x["img_shapes"]}, opt, noise=x["noise"], u=x["u"])
                gs.append(m.G32.clone())
        else:
            step = QwenImageEditStep(m, "mse", max_grad_norm=0.0, gradient_accumulation_steps=2)
            for it in range(3):
                for b in range(2):
                    emb = {**{k: x[k][b:b + 1] for k in keys}, "img_shapes": x["img_shapes"][b:b + 1]}
                    step.train_step(emb, opt, noise=x["noise"][b:b + 1], u=x["u"][b:b + 1])
                gs.append(m.G32.clone() / 2)  # the accumulator holds the SUM over micro-steps; the optimizer divides
            assert opt.step_count == 3
            n_graphs = step._graphs.captured()
            assert n_graphs == 2, f"expected one graph per micro-step kind, got {n_graphs}"
        out[mode] = (gs, [p.detach().float().clone() for p in m.parameters()])
    res = dict(grad=max(rel_l2(a, b) for a, b in zip(out["accum"][0], out["big"][0])))
    num = sum(((a - b) ** 2).sum() for a, b in zip(out["big"][1], out["accum"][1]))
    den = sum((a ** 2).sum() for a in out["big"][1])
    res["params_after_3_steps"] = float((num / den).sqrt())
    res["err"] = max(res["grad"], res["params_after_3_steps"])
    return res


def qwen_reference_rope_placement():
    """`rope_placement="reference"` on the CUDA path vs the oracle's restatement of transformer_qwen_custom.py:199-208 with padded text."""
    orc, m = build_pair(2, 2, 128, 4, ("to_q", "to_k", "to_v", "to_out.0"))
    g = torch.Generator(device="cuda").manual_seed(13)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g).bfloat16()
    shapes = [[(1, 8, 8), (1, 8, 8)], [(1, 4, 8), (1, 4, 8)]]
    T, txt = 24, [24, 13]
    pe = rn(2, T, 128) * 3
    pe[1, 13:] = 0
    mask = torch.zeros(2, T, dtype=torch.int64, device="cuda")
    mask[0], mask[1, :13] = 1, 1
    packed = torch.zeros(2, 128, 64, dtype=torch.bfloat16, device="cuda")
    packed[0], packed[1, :64] = rn(128, 64), rn(64, 64)
    sig = torch.tensor([0.5, 0.25], device="cuda")
    am = torch.zeros(2, T + 128, dtype=torch.bool, device="cuda")
    am[0], am[1, :13], am[1, T:T + 64] = True, True, True
    res = {}
    with torch.no_grad():
        for place in ("aligned", "reference"):
            ref = orc(hidden_states=packed.float(), timestep=sig, encoder_hidden_states=pe.float(), img_shapes=shapes, txt_seq_lens=txt,
                      attention_mask=am, img_offset=place)[0]
            m.rope_placement = place
            out = m(hidden_states=packed, timestep=sig, encoder_hidden_states=pe, encoder_hidden_states_mask=mask, img_shapes=shapes,
                    txt_seq_lens=txt)[0]
            res[place] = rel_l2(out.float(), ref)
            res[place + "_pad_rows_max"] = float(out[1, 64:].abs().max())
            if place == "aligned":
                ref_a = ref
        res["placements_differ"] = rel_l2(ref[1], ref_a[1])
    m.rope_placement = "aligned"
    assert res["placements_differ"] > 2e-2
    res["err"] = max(res["aligned"], res["reference"], res["aligned_pad_rows_max"], res["reference_pad_rows_max"])
    return res


def infer_graph_replay():
    """The no-grad forward replays a CUDA graph from its third call of a shape on: outputs must equal the eager forward bit for bit (no
    atomics on that path), for two alternating prompt lengths (true CFG: prompt / negative prompt), interleaved with a training step
    that uses another workspace, and for the whole sampling loop."""
    from qflux_b200.sampler import sample_qwen
    from qflux_b200.train_step import QwenImageEditStep
    orc, m = build_pair(2, 2, 128, 4, ("to_q", "to_k", "to_v", "to_out.0"))
    x = inputs(2, 4, 24, 128)
    g = torch.Generator(device="cuda").manual_seed(5)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g).bfloat16()
    packed = torch.cat([x["image_latents"], x["control_latents"]], 1)
    shapes = x["img_shapes"]

    def call(pe, hs, t):
        with torch.no_grad():
            return m(hidden_states=hs, timestep=torch.tensor([t, t], device="cuda"), encoder_hidden_states=pe,
                     encoder_hidden_states_mask=torch.ones(2, pe.shape[1], dtype=torch.int64, device="cuda"), img_shapes=shapes)[0].clone()
    pe_a, pe_b = x["prompt_embeds"], rn(2, 17, 128) * 3
    m.use_cuda_graph_inference = False
    ref = [call(pe_a, packed, 0.5), call(pe_b, packed, 0.5), call(pe_a, packed * 0.5, 0.25), call(pe_b, packed * 0.5, 0.25)]
    m.use_cuda_graph_inference = True
    worst = 0.0
    step = QwenImageEditStep(m)
    emb = {k: x[k] for k in ("image_latents", "control_latents", "prompt_embeds", "img_shapes")}
    for rep in range(4):  # 1st: warm, 2nd: capture + replay, then replays; a training step in between re-points the model's workspace
        got = [call(pe_a, packed, 0.5), call(pe_b, packed, 0.5), call(pe_a, packed * 0.5, 0.25), call(pe_b, packed * 0.5, 0.25)]
        worst = max(worst, max(float((a.float() - b.float()).abs().max()) for a, b in zip(got, ref)))
        if rep == 2:
            step.train_step(emb, noise=x["noise"], u=x["u"])
    n_graphs = m._infer_graphs.captured()
    assert n_graphs == 2, f"expected two captured inference graphs, got {n_graphs}"
    # the sampling loop end to end, graphed vs eager
    e = dict(latents=rn(2, 16, 64), control_latents=x["control_latents"], prompt_embeds=pe_a, prompt_embeds_mask=torch.ones(2, 24, dtype=torch.int64, device="cuda"),
             negative_prompt_embeds=pe_b, negative_prompt_embeds_mask=torch.ones(2, 17, dtype=torch.int64, device="cuda"), img_shapes=shapes,
             num_inference_steps=4, true_cfg_scale=3.0)
    out_g = sample_qwen(m, e)
    m.use_cuda_graph_inference = False
    out_e = sample_qwen(m, e)
    m.use_cuda_graph_inference = True
    res = dict(forward_max_abs=worst, sampler_max_abs=float((out_g.float() - out_e.float()).abs().max()), graphs=n_graphs)
    res["err"] = max(res["forward_max_abs"], res["sampler_max_abs"])
    return res


FLUX_YAML_TARGETS = (
    r"(.*x_embedder|.*transformer_blocks\.[0-9]+\.(norm|norm1)\.linear|.*transformer_blocks\.[0-9]+\.attn\.(to_k|to_q|to_v|to_add_out)"
    r"|.*transformer_blocks\.[0-9]+\.attn\.to_out\.0|.*single_transformer_blocks\.[0-9]+\.attn\.to_out"
    r"|.*single_transformer_blocks\.[0-9]+\.(proj_mlp|proj_out)|.*(?<!single_)transformer_blocks\.[0-9]+\.ff\.net\.2"
    r"|.*(?<!single_)transformer_blocks\.[0-9]+\.ff\.net\.0\.proj|.*(?<!single_)transformer_blocks\.[0-9]+\.norm1_context\.linear"
    r"|.*(?<!single_)transformer_blocks\.[0-9]+\.ff_context\.net\.0\.proj|.*(?<!single_)transformer_blocks\.[0-9]+\.ff_context\.net\.2"
    r"|.*(?<!single_)transformer_blocks\.[0-9]+\.attn\.(to_add_out|add_k_proj|add_q_proj|add_v_proj))")


def build_flux_pair(H=2, L=2, Ls=2, J=64, Pp=64, r=4, targets=("to_q", "to_k", "to_v", "to_out.0"), guidance=True):
    from oracle import mmdit_oracle as mo
    from qflux_b200.flux_model import FluxB200, FluxB200Config
    kw = dict(num_layers=L, num_single_layers=Ls, attention_head_dim=128, num_attention_heads=H, joint_attention_dim=J,
              pooled_projection_dim=Pp, guidance_embeds=guidance)
    orc = mo.init_synthetic_(mo.FluxOracle(mo.FluxConfig(**kw)), std=0.05 if H < 8 else 0.02)
    g = torch.Generator().manual_seed(98)
    with torch.no_grad():
        for n, p in orc.named_parameters():
            if n.endswith("bias"):
                p.copy_(torch.randn(p.shape, generator=g) * 0.02)
            elif p.ndim == 1:
                p.copy_(1 + torch.randn(p.shape, generator=g) * 0.1)
    mo.add_lora_adapter(orc, r=r, alpha=r, target_modules=targets, b_std=0.05)
    orc = orc.cuda()
    with torch.no_grad():
        for p in orc.parameters():
            p.copy_(p.bfloat16().float())
    m = FluxB200(FluxB200Config(**kw)).add_adapter(r, r, target_modules=targets)
    missing, unexpected = m.load_state_dict(orc.state_dict(), strict=True)
    assert not missing and not unexpected
    return orc, m


def flux_step_parity(H=2, L=2, Ls=2, J=64, Pp=64, B=2, hw=4, T=8, r=4,
                     targets=("to_q", "to_k", "to_v", "to_out.0"), guidance=True):
    """FLUX-Kontext shared-resolution recipe (flux_kontext_trainer.py:494-577) vs the oracle."""
    from oracle import mmdit_oracle as mo
    from qflux_b200.train_step import FluxKontextStep
    orc, m = build_flux_pair(H, L, Ls, J, Pp, r, targets, guidance)
    gg = torch.Generator(device="cuda").manual_seed(3)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=gg).bfloat16()
    Lt = hw * hw
    emb = dict(image_latents=rn(B, Lt, 64), control_latents=rn(B, Lt, 64), pooled_prompt_embeds=rn(B, Pp), prompt_embeds=rn(B, T, J),
               text_ids=torch.zeros(T, 3, device="cuda"), image_ids=FluxKontextStep.latent_image_ids(hw, hw, "cuda", 0.0),
               control_ids=FluxKontextStep.latent_image_ids(hw, hw, "cuda", 1.0))
    noise, t = rn(B, Lt, 64), torch.tensor([0.5, 0.25, 0.75, 0.125][:B], device="cuda")
    f = lambda k: emb[k].float()
    loss_o, pred_o = mo.flux_compute_loss_shared(orc, f("image_latents"), f("control_latents"), f("pooled_prompt_embeds"),
                                                 f("prompt_embeds"), emb["text_ids"], emb["image_ids"], emb["control_ids"],
                                                 noise=noise.float(), t=t)
    loss_o.backward()
    g_o = {n: (p.grad.clone() if p.grad is not None else torch.zeros_like(p)) for n, p in orc.named_parameters() if p.requires_grad}
    step = FluxKontextStep(m)
    loss_b = step.compute_loss(emb, noise=noise, t=t)
    pred_b = m._ws["pred"].view(B, -1, 64)[:, :Lt].float().clone()
    loss_b.backward()
    torch.cuda.synchronize()
    res = dict(pred_vs_fp32=rel_l2(pred_b, pred_o), loss=loss_o.item(), loss_abs=abs(loss_b.item() - loss_o.item()))
    res["loss_rel"] = res["loss_abs"] / max(1.0, abs(loss_o.item()))
    gb = {n: p.grad.float() for n, p in m.named_parameters()}
    num = sum(((gb[n] - g_o[n]).double() ** 2).sum() for n in g_o)
    den = sum((g_o[n].double() ** 2).sum() for n in g_o)
    res["grad_vs_fp32"] = float((num / den).sqrt())
    step.train_step(emb, noise=noise, t=t)
    gv = m.lora_grad_views()
    res["fast_vs_autograd"] = max(rel_l2(gv[n], gb[n]) for n in gb if gb[n].abs().max() > 0)
    orc.zero_grad()
    orc16 = orc.bfloat16()
    with eager_sdpa():  # not cuDNN attention: its backward is wrong for this oracle (lora_grad_check.eager_sdpa)
        loss_h, pred_h = mo.flux_compute_loss_shared(orc16, emb["image_latents"], emb["control_latents"], emb["pooled_prompt_embeds"],
                                                     emb["prompt_embeds"], emb["text_ids"], emb["image_ids"], emb["control_ids"],
                                                     noise=noise, t=t.bfloat16())
        loss_h.backward()
    g_h = {n: (p.grad.float() if p.grad is not None else torch.zeros_like(p).float()) for n, p in orc16.named_parameters() if p.requires_grad}
    res["bf16oracle_pred_vs_fp32"] = rel_l2(pred_h.float(), pred_o)
    _grad_per_tensor(res, gb, g_o, g_h)
    res["err"] = max(res["pred_vs_fp32"], res["grad_vs_fp32"])
    return res


def qwen_multires(H=2, L=2, J=128, shapes=None, expect_bands=False):
    """pad-to-max multi-resolution batch (per-sample RoPE, text + image key masks, AttentionMask loss) vs un-padded oracle runs.
    expect_bands: the shapes are large enough that the block GEMMs run on ragged row bands (lib.RowBands) and zero-fill the rest."""
    from oracle import mmdit_oracle as mo
    from qflux_b200.train_step import QwenImageEditStep
    orc, m = build_pair(H, L, J, 4, ("to_q", "to_k", "to_v", "to_out.0"))
    g = torch.Generator(device="cuda").manual_seed(11)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g).bfloat16()
    shapes = shapes or [[(1, 16, 12), (1, 16, 12)], [(1, 8, 10), (1, 8, 10)], [(1, 12, 12), (1, 12, 12)]]
    lt = [sh[0][1] * sh[0][2] for sh in shapes]
    lc = lt
    B, T, txt = 3, 40, [40, 23, 31]
    Lt = max(lt)
    x0, ctrl, pe, noise = rn(B, Lt, 64), rn(B, Lt, 64), rn(B, T, J) * 3, rn(B, Lt, 64)
    mask = torch.zeros(B, T, dtype=torch.int64, device="cuda")
    for b in range(B):
        x0[b, lt[b]:] = 0; ctrl[b, lc[b]:] = 0; noise[b, lt[b]:] = 0; pe[b, txt[b]:] = 0; mask[b, :txt[b]] = 1
    u = torch.tensor([0.5, 0.25, 0.75])
    sig = ((1000 - (u * 1000).long()).float() / 1000).cuda()
    preds, total = [], 0.0
    for b in range(B):
        s = sig[b]
        noisy = (1 - s) * x0[b, :lt[b]].float() + s * noise[b, :lt[b]].float()
        packed = torch.cat([noisy, ctrl[b, :lc[b]].float()], 0)[None]
        p = orc(hidden_states=packed, timestep=sig[b:b + 1], encoder_hidden_states=pe[b:b + 1, :txt[b]].float(),
                encoder_hidden_states_mask=mask[b:b + 1, :txt[b]], img_shapes=[shapes[b]], txt_seq_lens=[txt[b]])[0][0, :lt[b]]
        preds.append(p)
        total = total + ((p - (noise[b, :lt[b]].float() - x0[b, :lt[b]].float())) ** 2).mean(-1).sum()
    loss_o = total / (sum(lt) + 1e-12)
    loss_o.backward()
    step = QwenImageEditStep(m, "attention_mask")
    emb = dict(image_latents=x0, control_latents=ctrl, prompt_embeds=pe, prompt_embeds_mask=mask, img_shapes=shapes)
    loss_b = step.compute_loss(emb, noise=noise, u=u)
    pred_b = m._ws["pred"].view(B, -1, 64).float().clone()
    loss_b.backward()
    torch.cuda.synchronize()
    res = dict(pred_vs_fp32=max(rel_l2(pred_b[b, :lt[b]], preds[b]) for b in range(B)), loss=loss_o.item(),
               loss_abs=abs(loss_b.item() - loss_o.item()))
    res["loss_rel"] = res["loss_abs"] / max(1.0, abs(loss_o.item()))
    go = {n: p.grad for n, p in orc.named_parameters() if p.requires_grad}
    num = sum(((p.grad.float() - go[n]).double() ** 2).sum() for n, p in m.named_parameters())
    den = sum((v.double() ** 2).sum() for v in go.values())
    res["grad_vs_fp32"] = float((num / den).sqrt())
    res["err"] = max(res["pred_vs_fp32"], res["grad_vs_fp32"])
    bands = m._ws.get("bands")
    res["bands"] = None if bands is None else dict(n=bands.n, dead=bands.host_dead)
    if expect_bands:
        assert bands is not None and bands.n_dead > 0, "the ragged GEMM path was not taken"
    return res


def flux_multires(H=2, L=2, Ls=2, J=64, Pp=64, shapes=None, expect_bands=False):
    """FLUX pad-to-max multi-resolution recipe (flux_kontext_trainer.py:579-796): per-sample ids / RoPE, key mask, masked loss —
    against one un-padded oracle run per sample."""
    from qflux_b200.train_step import FluxKontextStep
    orc, m = build_flux_pair(H, L, Ls, J, Pp, 4, r".*(attn\.to_[qkv]|to_out\.0|proj_mlp|single_transformer_blocks\.[0-9]+\.proj_out)")
    g = torch.Generator(device="cuda").manual_seed(21)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g).bfloat16()
    shapes = shapes or [[(1, 16, 12), (1, 16, 12)], [(1, 8, 10), (1, 10, 8)], [(1, 12, 8), (1, 6, 8), (1, 8, 12)]]
    B, T = 3, 24
    lt = [sh[0][1] * sh[0][2] for sh in shapes]
    lc = [sum(h * w for (_, h, w) in sh[1:]) for sh in shapes]
    Lm, Lcm = max(lt), max(lc)
    x0, ctrl, noise = rn(B, Lm, 64), rn(B, Lcm, 64), rn(B, Lm, 64)
    for b in range(B):
        x0[b, lt[b]:] = 0; noise[b, lt[b]:] = 0; ctrl[b, lc[b]:] = 0
    pe, pooled, t = rn(B, T, J), rn(B, Pp), torch.tensor([0.5, 0.25, 0.125], device="cuda")
    text_ids = torch.zeros(T, 3, device="cuda")
    preds, total = [], 0.0
    for b in range(B):
        ids = [FluxKontextStep.latent_image_ids(shapes[b][0][1], shapes[b][0][2], "cuda", 0.0)]
        ids += [FluxKontextStep.latent_image_ids(h, w, "cuda", float(j + 1)) for j, (_, h, w) in enumerate(shapes[b][1:])]
        noisy = (1 - t[b]) * x0[b, :lt[b]].float() + t[b] * noise[b, :lt[b]].float()
        packed = torch.cat([noisy.bfloat16().float(), ctrl[b, :lc[b]].float()], 0)[None]
        p = orc(hidden_states=packed, encoder_hidden_states=pe[b:b + 1].float(), pooled_projections=pooled[b:b + 1].float(),
                timestep=t[b:b + 1], img_ids=torch.cat(ids, 0), txt_ids=text_ids, guidance=torch.ones(1, device="cuda"))[0][0, :lt[b]]
        preds.append(p)
        total = total + ((p - (noise[b, :lt[b]].float() - x0[b, :lt[b]].float())) ** 2).mean(-1).sum()
    loss_o = total / (sum(lt) + 1e-12)
    loss_o.backward()
    step = FluxKontextStep(m, "attention_mask")
    emb = dict(image_latents=x0, control_latents=ctrl, pooled_prompt_embeds=pooled, prompt_embeds=pe, text_ids=text_ids, img_shapes=shapes)
    loss_b = step.compute_loss(emb, noise=noise, t=t)
    pred_b = m._ws["pred"].view(B, -1, 64).float().clone()
    loss_b.backward()
    torch.cuda.synchronize()
    res = dict(pred_vs_fp32=max(rel_l2(pred_b[b, :lt[b]], preds[b]) for b in range(B)), loss=loss_o.item(),
               loss_abs=abs(loss_b.item() - loss_o.item()))
    res["loss_rel"] = res["loss_abs"] / max(1.0, abs(loss_o.item()))
    go = {n: (p.grad if p.grad is not None else torch.zeros_like(p)) for n, p in orc.named_parameters() if p.requires_grad}
    num = sum(((p.grad.float() - go[n]).double() ** 2).sum() for n, p in m.named_parameters())
    den = sum((v.double() ** 2).sum() for v in go.values())
    res["grad_vs_fp32"] = float((num / den).sqrt())
    res["err"] = max(res["pred_vs_fp32"], res["grad_vs_fp32"])
    bands = m._ws.get("bands")
    res["bands"] = None if bands is None else dict(n=bands.n, dead=bands.host_dead)
    if expect_bands:
        assert bands is not None and bands.n_dead > 0, "the ragged GEMM path was not taken"
    return res


def sampler_tiny():
    """Euler / true-CFG sampling loops (qflux_b200/sampler.py) on the fused forward against the same loop driven by the fp32 oracle."""
    from qflux_b200 import sampler
    from qflux_b200.train_step import FluxKontextStep

    class F32:  # the oracle behind the module signature, bf16 in / bf16 out like a bf16 model
        def __init__(self, net):
            self.net, self.device = net, torch.device("cuda")

        def __call__(self, **kw):
            if "pooled_projections" in kw:  # a bf16 FLUX model multiplies timestep / guidance by 1000 in bf16 (transformer_flux.py:707-710)
                for k in ("timestep", "guidance"):
                    kw[k] = (kw[k].bfloat16() * 1000).float() / 1000
            kw = {k: (v.float() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in kw.items()}
            if "txt_seq_lens" in kw and kw["txt_seq_lens"] is None:
                kw["txt_seq_lens"] = kw["encoder_hidden_states_mask"].sum(1).tolist()
            with torch.no_grad():
                return (self.net(**kw)[0].bfloat16(),)

    g = torch.Generator(device="cuda").manual_seed(5)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g).bfloat16()
    B, hw, T = 2, 8, 24
    orc, m = build_pair(2, 2, 128, 4, ("to_q", "to_k", "to_v", "to_out.0"))
    emb = dict(latents=rn(B, hw * hw, 64), control_latents=rn(B, hw * hw, 64), prompt_embeds=rn(B, T, 128) * 3,
               prompt_embeds_mask=torch.ones(B, T, dtype=torch.int64, device="cuda"), negative_prompt_embeds=rn(B, T, 128) * 3,
               negative_prompt_embeds_mask=torch.ones(B, T, dtype=torch.int64, device="cuda"), img_shapes=[[(1, hw, hw), (1, hw, hw)]] * B,
               num_inference_steps=4, true_cfg_scale=2.5)
    res = dict(qwen=rel_l2(sampler.sample_qwen(m, emb).float(), sampler.sample_qwen(F32(orc), emb).float()))
    forc, fm = build_flux_pair()
    femb = dict(latents=rn(B, hw * hw, 64), latent_ids=FluxKontextStep.latent_image_ids(hw, hw, "cuda", 0.0),
                control_latents=rn(B, hw * hw, 64), control_ids=FluxKontextStep.latent_image_ids(hw, hw, "cuda", 1.0),
                pooled_prompt_embeds=rn(B, 64), prompt_embeds=rn(B, T, 64), text_ids=torch.zeros(T, 3, device="cuda"), guidance=3.5,
                negative_pooled_prompt_embeds=rn(B, 64), negative_prompt_embeds=rn(B, T, 64), negative_text_ids=torch.zeros(T, 3, device="cuda"),
                num_inference_steps=4, true_cfg_scale=1.5)
    res["flux"] = rel_l2(sampler.sample_flux(fm, femb).float(), sampler.sample_flux(F32(forc), femb).float())
    res["err"] = max(res.values())
    return res


CASES = {
    "inference_tiny": inference_parity,
    "step_tiny": lambda: step_parity(),
    "step_tiny_nolora_targets_all_attn": lambda: step_parity(targets=("to_q", "to_k", "to_v", "to_out.0", "add_q_proj", "add_k_proj", "add_v_proj", "to_add_out", "net.0.proj"), r=8),
    "step_mid": lambda: step_parity(H=4, L=3, J=256, B=2, hw=16, T=40, r=16),
    "step_full_width_1blk": full_width_block,
    "qwen_multires": qwen_multires,
    "flux_tiny": lambda: flux_step_parity(),
    "flux_tiny_regex_noguidance": lambda: flux_step_parity(guidance=False, r=8,
                                                           targets=r".*(attn\.(to_[qkv]|add_[qkv]_proj|to_add_out)|proj_mlp|ff\.net\.0\.proj)"),
    "flux_tiny_mlp_out_targets": lambda: flux_step_parity(
        r=8, targets=r".*(single_transformer_blocks\.[0-9]+\.(proj_mlp|proj_out)|ff\.net\.2|ff_context\.net\.(0\.proj|2)|attn\.to_out\.0)"),
    "flux_multires": flux_multires,
    # the same recipes with image sizes whose padding spans whole 256-row GEMM bands: ragged row bands + zero fill on the product path
    "qwen_multires_bands": lambda: qwen_multires(shapes=[[(1, 32, 24), (1, 32, 24)], [(1, 12, 10), (1, 12, 10)], [(1, 20, 20), (1, 20, 20)]],
                                                 expect_bands=True),
    "flux_multires_bands": lambda: flux_multires(shapes=[[(1, 32, 24), (1, 32, 24)], [(1, 8, 10), (1, 10, 8)], [(1, 20, 16), (1, 12, 8), (1, 16, 20)]],
                                                 expect_bands=True),
    "sampler_tiny": sampler_tiny,
    # BASELINE config 3 target set (configs/face_seg_flux_kontext_fp16.yaml:11): every block Linear, the AdaLN linears, x_embedder
    "flux_tiny_yaml_targets": lambda: flux_step_parity(r=8, targets=FLUX_YAML_TARGETS),
    "step_tiny_mod_embed_targets": lambda: step_parity(targets=("to_q", "img_mod.1", "txt_mod.1", "img_in", "txt_in")),
    "step_tiny_mlp_down_targets": lambda: step_parity(targets=("to_k", "img_mlp.net.2", "txt_mlp.net.0.proj", "txt_mlp.net.2")),
    "flux_full_width_1p1": lambda: flux_step_parity(H=24, L=1, Ls=1, J=4096, Pp=768, B=1, hw=32, T=512, r=16),
    "bench_point_6blk": bench_point_6blk,
    "infer_graph_replay": infer_graph_replay,
    "grad_accum": grad_accum,
    "qwen_reference_rope_placement": qwen_reference_rope_placement,
    "train_trajectory_5steps": train_trajectory,
    "graph_replay": graph_replay,
}

if __name__ == "__main__":
    main(CASES, os.path.abspath(__file__), "model_check.log")
