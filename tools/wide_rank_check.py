"""GPU check of LoRA ranks above 64 (the factors padded to Rp = 128, two 64-wide k-blocks):

  wgrad_tc_*     qfx_lora_wgrad_tc and its _det twin per element against fp64 (reduce_check.py's bound, sentinels, NaN-filled scratch
                 of exactly lib.det_scratch_wgrad_tc, bitwise repeat of the twin) at r = 1, 24, 64, 68, 96, 128 with B's groups Rp wide,
                 modes 0 / 1, G = 1-3, M not a multiple of 64; B's columns in [r, Rp) of every group hold a large value;
  gemm_kb2       qfx_gemm_bf16 with two appended LoRA k-blocks per tile and row (gemm_tile_check.py): a plain problem, a q|k|v
                 lora_group_n problem (A2 columns g*128 ...) and the trans_b = 1 dgrads with kb2 = 2 and 6 (a three-slot site);
  det_graph_*    a Qwen (every Linear, img_in's chunked narrow path included) and a FLUX (BASELINE config 3's targets) training step
                 at r = 128 / 96: under torch.use_deterministic_algorithms(True) eager and CUDA-graph steps give bit-identical G32
                 step after step; with the flag off graph replays match the eager step within fp32 reordering;
  trajectory_r128  model_check.train_trajectory at r = 128: 5 fused AdamW steps against the fp32 oracle, loss within 1e-2.
Run stand-alone: `python tools/wide_rank_check.py [case ...]` (one subprocess per case)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from harness import ROOT, main  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import gemm_tile_check as gt  # noqa: E402
import reduce_check as rc  # noqa: E402
from glue_check import RED_TOL, Checks, _mk  # noqa: E402

WR_R = [1, 24, 64, 68, 96, 128]
WR_M = [65, 1000, 8191]


def wgrad_ref(A, B, r, G, mode=0, Dg=0):
    """per group g: (sum_m A[m, i] B[m, g*Rp + j], sum_m |A B|), j < r, fp64"""
    rp = 64 * -(-r // 64)
    Ad, Bd = A.double(), B.double()
    out = []
    for g in range(G):
        a = Ad[:, g * Dg:(g + 1) * Dg] if mode == 1 else Ad
        b = Bd[:, g * rp:g * rp + r]
        out.append((a.t() @ b, a.abs().t() @ b.abs()))
    return out


def _one(c, mode, G, Dg, r, Na, M, layout, seed):
    from qflux_b200 import lib
    rp = 64 * -(-r // 64)
    tag = f"wgrad_tc mode{mode} G{G} r{r} Na{Na} M{M} {layout}"
    A = _mk(M, Na + 72, seed=seed)[:, 8:8 + Na]
    Bm = _mk(M, rp * G + 24, seed=seed + 1)[:, 8:8 + rp * G]
    for g in range(G):
        Bm[:, g * rp + r:(g + 1) * rp] = rc.BIG
    rows = Dg if mode == 1 else Na
    gs_i, gs_j = (r, 1) if layout == "dB" else (1, rows)
    refs = wgrad_ref(A, Bm, r, G, mode, Dg)
    inits = [rc._init(rows * r, seed + 10 + g) for g in range(G)]

    def outputs():
        s = rc.Slots([rows * r] * G)
        for g in range(G):
            s[g].copy_(inits[g])
        return s

    def view(t):
        return torch.as_strided(t, (rows, r), (gs_i, gs_j))

    def check(var, s):
        for g, (ref, mag) in enumerate(refs):
            i0 = view(inits[g]).double()
            rc._bound(c, f"wgrad_tc_{var}_max_err_over_bound", f"{tag} {var} group {g}", view(s[g]), i0 + ref, RED_TOL * (i0.abs() + mag))
        rc._sentinels(c, f"{tag} {var}", s.buf, s.free, rc.SENT)

    ng = 1 if mode == 1 else G
    rc._run_both(c, tag, lambda s: lib.lora_wgrad_tc(A, Bm, [s[g] for g in range(G)], gs_i, gs_j, r, mode=mode, Dg=Dg),
                 lambda s, scr: lib.lora_wgrad_tc_det(A, Bm, [s[g] for g in range(G)], gs_i, gs_j, r, mode=mode, Dg=Dg, scratch=scr),
                 lib.det_scratch_wgrad_tc(M, Na, ng, r), outputs, check)


def wgrad_sweep(mode, G, Dg=0):
    c = Checks()
    k = 0
    for r in WR_R:
        for j, M in enumerate(WR_M):
            Na = G * Dg if mode == 1 else (128, 3072, 384)[(k + G) % 3]
            _one(c, mode, G, Dg, r, Na, M, ("dB", "dA")[k % 2], seed=100 * k + 17)
            k += 1
    c.res["cases"] = k
    return c.out()


def gemm_kb2():
    c = Checks()
    p = gt._prob(1000, 384, 3072, False, 1, kb2=2, bias=True)                                     # one adapted projection, Rp = 128
    gt.run(c, "plain", [p], 384, 3072, trans_b=False, epi=gt.EPI_BIAS, bn=128)
    probs = [gt._prob(1000, 384, 256, False, 3, kb2=2, groups=3, bias=True), gt._prob(129, 384, 256, False, 5, kb2=2, groups=3)]
    gt.run(c, "qkv", probs, 384, 256, trans_b=False, epi=gt.EPI_BIAS, bn=128, lora_group_n=128)  # A2 columns g*128 + j*64
    for kb2 in (2, 6):                                                                             # one slot / a q|k|v site's three slots
        probs = [gt._prob(1000, 256, 768, True, 7, kb2=kb2), gt._prob(77, 256, 768, True, 9, kb2=kb2)]
        gt.run(c, f"dgrad_kb{kb2}", probs, 256, 768, trans_b=True, epi=gt.EPI_BIAS, alpha=0.5, bn=128)
    return c.out()


def _model(kind, r):
    import lora_grad_check as lg
    from qflux_b200.train_step import FluxKontextStep, QwenImageEditStep
    g = torch.Generator().manual_seed(5)
    rn = lambda *s: torch.randn(*s, generator=g).bfloat16().cuda()
    B, hw, T = 2, 8, 24
    if kind == "qwen":
        _, m = lg.qwen_pair(torch.device("cuda"), r=r)
        emb = dict(image_latents=rn(B, hw * hw, 64), control_latents=rn(B, hw * hw, 64), prompt_embeds=rn(B, T, m.J) * 3,
                   img_shapes=[[(1, hw, hw), (1, hw, hw)]] * B)
        kw = dict(noise=rn(B, hw * hw, 64), u=torch.tensor([0.5, 0.25]))
        return m, lambda graph: QwenImageEditStep(m, use_cuda_graph=graph), emb, kw
    _, m = lg.flux_pair(torch.device("cuda"), r=r, targets=lg._flux_yaml_targets())
    emb = dict(image_latents=rn(B, hw * hw, 64), control_latents=rn(B, hw * hw, 64), pooled_prompt_embeds=rn(B, 64),
               prompt_embeds=rn(B, T, 64), text_ids=torch.zeros(T, 3),
               image_ids=FluxKontextStep.latent_image_ids(hw, hw, "cpu", 0.0), control_ids=FluxKontextStep.latent_image_ids(hw, hw, "cpu", 1.0))
    kw = dict(noise=rn(B, hw * hw, 64), t=torch.tensor([0.5, 0.25]))
    return m, lambda graph: FluxKontextStep(m, use_cuda_graph=graph), emb, kw


def det_graph(kind, r):
    """G32 after an eager step and after three steps of a graphed step object (warm-up, capture, replay), flag on and off"""
    c = Checks()
    m, make, emb, kw = _model(kind, r)
    c.res["rank"], c.res["rp"], c.res["n_grad"] = m.lora_rank, m.lora_rp, m.G32.numel()
    for det in (True, False):
        torch.use_deterministic_algorithms(det)
        losses, gs = [float(make(False).train_step(emb, **kw))], [m.G32.clone()]
        graphed = make(True)
        for _ in range(3):
            losses.append(float(graphed.train_step(emb, **kw)))
            gs.append(m.G32.clone())
        torch.cuda.synchronize()
        tag = "det" if det else "atomic"
        c.res[f"{tag}_losses"] = losses
        c.check(all(torch.isfinite(g).all() for g in gs) and gs[0].abs().sum() > 0, f"{tag}: non-finite or zero gradient")
        if det:
            for i in range(1, 4):
                c.check(torch.equal(gs[i].view(torch.int32), gs[0].view(torch.int32)), f"det: step {i} G32 differs from the eager step's")
                c.check(losses[i] == losses[0], f"det: step {i} loss {losses[i]!r} != {losses[0]!r}")
        else:
            worst = max(float((g - gs[0]).norm() / gs[0].norm()) for g in gs[1:])
            c.res["atomic_max_rel"] = worst
            c.check(worst < 1e-4, f"atomic: graph replay differs from the eager step by rel-L2 {worst:.3g}")
    c.res["graphs_captured"] = True
    return c.out()


def trajectory_r128():
    import model_check
    c = Checks()
    r = model_check.train_trajectory(r=128)
    c.res.update(r)
    c.check(r["err"] < 1e-2, f"loss trajectory off the oracle by {r['err']:.3g}")
    c.check(r["decreased"], "loss did not decrease")
    return c.out()


CASES = {}
for _G in (1, 2, 3):
    CASES[f"wgrad_tc_mode0_G{_G}"] = (lambda G: lambda: wgrad_sweep(0, G))(_G)
for _G in (2, 3):
    for _Dg in (128, 3072):
        CASES[f"wgrad_tc_mode1_G{_G}_Dg{_Dg}"] = (lambda G, Dg: lambda: wgrad_sweep(1, G, Dg))(_G, _Dg)
CASES["gemm_kb2"] = gemm_kb2
CASES["det_graph_qwen_r128"] = lambda: det_graph("qwen", 128)
CASES["det_graph_flux_yaml_r96"] = lambda: det_graph("flux", 96)
CASES["trajectory_r128"] = trajectory_r128

if __name__ == "__main__":
    main(CASES, os.path.abspath(__file__), "wide_rank_check.log")
