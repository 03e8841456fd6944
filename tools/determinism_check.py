"""GPU checks of the deterministic training step (torch.use_deterministic_algorithms(True)), one subprocess per case:

    python tools/determinism_check.py [case ...]

Every case turns the flag on and runs with CUBLAS_WORKSPACE_CONFIG set (torch refuses the modulation-LoRA cuBLAS products under the
flag without it).

  attn_kernels         qfx_attn_bwd_det through every case of tools/attn_check.py (its fp64 per-(b, h, row) bounds, sentinels, exact
                       zeros, dQ accumulating into a prefilled buffer and leaving rows >= kv_len alone), then dQ, dK and dV
                       bit-identical across two launches at each of those shapes
  reductions           qfx_lora_wgrad_tc_det (mode 0 with three groups, mode 1), qfx_lora_wgrad_det, qfx_mod_grad_det,
                       qfx_flow_loss_det, qfx_grad_finalize_det, qfx_fused_adamw_det: bit-identical across two launches, and within
                       tools/glue_check.py's fp32-reduction bound of an fp64 reference (the atomic kernels are held to the same bound)
  r2r_*                three train_steps with FusedLoraAdamW from a fixed seed; returns SHA-256 digests of the losses, G32 and every
                       LoRA weight.  tests/test_deterministic_step.py runs each case in two processes and compares the digests
  graph_and_recompute  loss and G32 bit for bit: eager step vs CUDA-graph replay, every block kept vs blocks forced into recompute
                       (set_activation_memory_limit); also two inference forwards; and, reported without assertion, how many G32
                       elements two flag-off steps disagree on
  fp8_vs_bf16 / nf4_vs_bf16   loss, prediction and G32 bit for bit: FP8- / NF4-resident model vs a bf16 model holding the upcast /
                       dequantized weights
  lora_grad_<case>     tools/lora_grad_check.py's per-tensor fp64 bound with the fused model on the deterministic path (the eager
                       oracles run with the flag off: the check is about the fused kernels)
"""
import hashlib
import os
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "qwen-image-finetune_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import harness  # noqa: E402


def _det():
    import torch
    torch.use_deterministic_algorithms(True)
    return torch


def _sha(*ts):
    h = hashlib.sha256()
    for t in ts:
        h.update(t.detach().contiguous().view(-1).view(__import__("torch").uint8).cpu().numpy().tobytes())
    return h.hexdigest()


def _bits_equal(a, b):
    return a.shape == b.shape and bool((a.contiguous().view(-1).view(__import__("torch").uint8)
                                        == b.contiguous().view(-1).view(__import__("torch").uint8)).all())


# ================================================================================================================ kernels
def attn_kernels():
    torch = _det()
    import attn_check
    from gemm_tile_check import sentinel
    from qflux_b200 import lib
    lib.attn_bwd = lib.attn_bwd_det  # attn_check.run calls lib.attn_bwd: every case below runs the deterministic backward
    res, fail = {}, []
    shapes = {}
    real_run = attn_check.run

    def spy(c, B, H, S, split, txt=None, kv=None, **kw):
        shapes[(B, H, S, split)] = (txt, kv)
        return real_run(c, B, H, S, split, txt, kv, **kw)
    attn_check.run = spy
    for name, fn in attn_check.CASES.items():
        r = fn()
        res[name] = {k: v for k, v in r.items() if k.endswith("worst_over_eager") or k == "fail"}
        fail += [f"{name}: {f}" for f in r["fail"]]
    for (B, H, S, split), (txt, kv) in shapes.items():
        Q, K, V, dO = (attn_check._mk(B, H, S, 128, seed=10 + i, device="cuda") for i in range(4))
        kv_len = None if kv is None else torch.tensor(kv, dtype=torch.int32, device="cuda")
        txt_len = None if txt is None else torch.tensor(txt, dtype=torch.int32, device="cuda")
        ot, oi = torch.empty(B * split, H * 128, device="cuda", dtype=torch.bfloat16), torch.empty(B * (S - split), H * 128, device="cuda",
                                                                                                     dtype=torch.bfloat16)
        lse = torch.empty(B, H, S, device="cuda")
        lib.attn_fwd(Q, K, V, ot, oi, split, lse, kv_len, txt_len=txt_len)
        delta = torch.randn(B, H, S, device="cuda") * 0.1
        outs = []
        for _ in range(2):
            dq = torch.zeros(B, H, S, 128, device="cuda")
            dk, dv = sentinel(B, H, S, 128, device="cuda"), sentinel(B, H, S, 128, device="cuda")
            lib.attn_bwd_det(Q, K, V, dO, lse, delta, dq, dk, dv, kv_len, txt_len=txt_len, split=split)
            outs.append((dq, dk, dv))
        torch.cuda.synchronize()
        for nm, a, b in zip(("dQ", "dK", "dV"), outs[0], outs[1]):
            if not _bits_equal(a, b):
                fail.append(f"{nm} differs between two launches at B={B} H={H} S={S} split={split}")
    res["repeat_shapes"] = len(shapes)
    res["fail"] = fail
    assert not fail, fail[:5]
    return res


def reductions():
    torch = _det()
    from glue_check import RED_TOL, _mk, _up
    from qflux_b200 import lib
    fail, res = [], {}

    def twice(name, fn, outs, ref, mag):
        """fn() fills `outs` (zeroed / refilled by fn); two launches must agree bit for bit and stay within RED_TOL * mag of ref"""
        a = [o.clone() for o in fn()]
        b = [o.clone() for o in fn()]
        torch.cuda.synchronize()
        same = all(_bits_equal(x, y) for x, y in zip(a, b))
        err = max(((x.double().cpu() - r).abs() / (m + 1e-30)).max().item() for x, r, m in zip(a, ref, mag))
        res[name] = dict(bitwise_repeat=same, err_over_mag=err)
        if not same:
            fail.append(f"{name}: two launches differ")
        if not err <= RED_TOL:
            fail.append(f"{name}: error {err:.3g} of the magnitude exceeds {RED_TOL}")

    # lora_wgrad_tc: mode 0 with three groups (dA of a fused q|k|v site), mode 1 (dB), M past one split and ragged
    M, Na, r = 3000, 3072, 16
    A, Bm = _mk(M, Na, seed=1), _mk(M, 3 * 64, seed=2)
    scr = torch.empty(max(lib.det_scratch_wgrad_tc(M, Na, 3, r), lib.det_scratch_wgrad_tc(M, Na, 1, r)), device="cuda")
    Gs = [torch.empty(Na * r, device="cuda") for _ in range(3)]
    pre = torch.randn(Na * r, device="cuda")

    def wg0():
        for g in Gs:
            g.copy_(pre)
        lib.lora_wgrad_tc_det(A, Bm, Gs, r, 1, r, mode=0, scratch=scr)
        return Gs
    Ad, Bd = A.double().cpu(), Bm.double().cpu()
    ref0 = [pre.double().cpu() + (Ad.t() @ Bd[:, g * 64:g * 64 + r]).reshape(-1) for g in range(3)]
    mag0 = [pre.double().cpu().abs() + (Ad.abs().t() @ Bd[:, g * 64:g * 64 + r].abs()).reshape(-1) for g in range(3)]
    twice("lora_wgrad_tc_det_mode0", wg0, Gs, ref0, mag0)
    Dg = Na // 3

    def wg1():
        for g in Gs:
            g.copy_(pre)
        lib.lora_wgrad_tc_det(A, Bm, Gs, r, 1, r, mode=1, Dg=Dg, scratch=scr)
        return Gs
    ref1 = [pre.double().cpu()[:Dg * r] + (Ad[:, g * Dg:(g + 1) * Dg].t() @ Bd[:, g * 64:g * 64 + r]).reshape(-1) for g in range(3)]
    mag1 = [pre.double().cpu().abs()[:Dg * r] + (Ad[:, g * Dg:(g + 1) * Dg].abs().t() @ Bd[:, g * 64:g * 64 + r].abs()).reshape(-1)
            for g in range(3)]
    twice("lora_wgrad_tc_det_mode1", lambda: [g[:Dg * r] for g in wg1()], Gs, ref1, mag1)
    # lora_wgrad (CUDA cores, the 64-channel embedder): [64, r] transposed store (gs_i = 1, gs_j = Dp)
    P, Qm = _mk(2100, 64, seed=3), _mk(2100, 64, seed=4)
    G = torch.empty(64 * r, device="cuda")
    scr2 = torch.empty(lib.det_scratch_wgrad(2100, 64, r), device="cuda")

    def wgc():
        G.zero_()
        lib.lora_wgrad_det(P, Qm, G, 1, 64, r, scratch=scr2)
        return [G]
    Pd, Qd = P.double().cpu(), Qm.double().cpu()
    twice("lora_wgrad_det", wgc, [G], [(Pd.t() @ Qd[:, :r]).t().reshape(-1)], [(Pd.abs().t() @ Qd[:, :r].abs()).t().reshape(-1)])
    # mod_grad: d shift + d scale with the row statistics, B = 3 samples of 700 rows
    rpb, D = 700, 3072
    g, m = _mk(3 * rpb, D, seed=5), _mk(3 * rpb, D, seed=6)
    mean, rstd = m.float().mean(1), torch.rsqrt(m.float().var(1, unbiased=False) + 1e-6)
    so, po = torch.empty(3, D, device="cuda"), torch.empty(3, D, device="cuda")
    scr3 = torch.empty(lib.det_scratch_mod_grad(3 * rpb, rpb, D), device="cuda")

    def mg():
        so.fill_(0.25)
        po.fill_(-0.5)
        lib.mod_grad_det(g, rpb, sum_out=so, m=m, prod_out=po, mean=mean, rstd=rstd, scratch=scr3)
        return [so, po]
    gv = g.double().cpu().view(3, rpb, D)
    mh = ((m.float() - mean[:, None]) * rstd[:, None]).to(torch.bfloat16).double().cpu().view(3, rpb, D)
    twice("mod_grad_det", mg, [so, po], [0.25 + gv.sum(1), -0.5 + (gv * mh).sum(1)],
          [0.25 + gv.abs().sum(1), 0.5 + (gv * mh).abs().sum(1) + (_up(mh) * gv.abs()).sum(1) / RED_TOL])
    # flow_loss
    B, L, Cc = 2, 4096, 64
    x0, noise, pred = _mk(B, L, Cc, seed=7), _mk(B, L, Cc, seed=8), _mk(B, 2 * L, Cc, seed=9)
    wt = torch.rand(B, L, device="cuda") + 0.5
    norm = 1.0 / (B * L * Cc)
    loss, dpred = torch.empty(1, device="cuda"), torch.empty_like(pred)
    scr4 = torch.empty(lib.DET_NORM_PARTIALS, device="cuda")

    def fl():
        lib.flow_loss_det(pred, x0, noise, wt, norm, loss, dpred, scratch=scr4)
        return [loss]
    tgt = (noise.double() - x0.double()).to(torch.bfloat16).double()
    d2 = wt.double()[..., None] * (pred[:, :L].double() - tgt) ** 2
    twice("flow_loss_det", fl, [loss], [(d2.sum() * norm).reshape(1).cpu()], [(d2.sum() * norm).reshape(1).cpu()])
    # grad_finalize / fused_adamw norms over a LoRA-sized gradient
    n = 5_000_000
    gg = _mk(n, seed=10, dtype=torch.float32)
    ss, ob = torch.empty(1, device="cuda"), torch.empty(n, device="cuda", dtype=torch.bfloat16)
    ref_ss = (gg.double() * 0.5).pow(2).sum().reshape(1).cpu()

    def gf():
        lib.grad_finalize_det(gg, 0.5, 1.0, ss, ob, scratch=scr4)
        return [ss]
    twice("grad_finalize_det", gf, [ss], [ref_ss], [ref_ss])
    p = torch.zeros(n // 1000, 1000, device="cuda", dtype=torch.bfloat16)
    tables = lib.adamw_tables([(p, 0)], "cuda")
    ea, eas, ss2 = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda"), torch.empty(1, device="cuda")

    def aw():
        p.zero_(), ea.zero_(), eas.zero_()
        lib.fused_adamw_det(tables, gg, ea, eas, ss2, 0.5, 1.0, 1e-4, 0.9, 0.999, 1e-8, 0.01, 1, scratch=scr4)
        return [ss2, p.float().view(-1)]
    a1 = [t.clone() for t in aw()]
    a2 = [t.clone() for t in aw()]
    res["fused_adamw_det"] = dict(bitwise_repeat=all(_bits_equal(x, y) for x, y in zip(a1, a2)),
                                  err_over_mag=((a1[0].double().cpu() - ref_ss).abs() / ref_ss).item())
    if not res["fused_adamw_det"]["bitwise_repeat"]:
        fail.append("fused_adamw_det: two launches differ")
    if not res["fused_adamw_det"]["err_over_mag"] <= RED_TOL:
        fail.append("fused_adamw_det: norm beyond the reduction bound")
    res["fail"] = fail
    assert not fail, fail
    return res


# ================================================================================================================ training steps
def _build(family, name, **over):
    import bench
    import fp8_check
    cfg = dict(bench.CONFIGS[name], **over)
    return fp8_check.build(family, cfg, fp8=False), cfg


def _batch(cfg, name, family, txt=None):
    import nf4_check
    b = nf4_check._fixed(nf4_check.device_batch(cfg, name), family)
    if txt is not None:  # a ragged prompt mask: sample b keeps its first txt[b] text tokens
        mask = b["prompt_embeds_mask"].clone()
        for i, t in enumerate(txt):
            mask[i, t:] = 0
        b["prompt_embeds_mask"] = mask
    return b


def _three_steps(family, name, txt=None, **over):
    torch = _det()
    import nf4_check
    from qflux_b200.optim import FusedLoraAdamW
    torch.manual_seed(0)
    m, cfg = _build(family, name, **over)
    batch = _batch(cfg, name, family, txt)
    step = nf4_check._step(m, family)
    opt = FusedLoraAdamW(m, lr=1e-3)
    losses = []
    for _ in range(3):
        losses.append(step.train_step(batch, opt, batch["noise"], batch["u"] if family == "qwen" else batch["timestep"]).clone())
    torch.cuda.synchronize()
    assert m._ws["det"] and "det_scratch" in m._ws
    w = [p for _, p in sorted(m._lora_params.items())]
    return dict(losses=[float(x) for x in losses], loss_sha=_sha(*losses), g32_sha=_sha(m.G32), lora_sha=_sha(*w), n_lora=len(w),
                graphs=step._graphs.captured(), gpu=torch.cuda.get_device_name())


def graph_and_recompute():
    torch = _det()
    import nf4_check
    m, cfg = _build("qwen", "qwen_edit", B=2, blocks=4)
    batch = _batch(cfg, "qwen_edit", "qwen")
    step = nf4_check._step(m, "qwen")
    args = step._prepare(batch, batch["noise"], batch["u"])
    outs = []
    for _ in range(3):  # eager, capture + first replay, replay
        outs.append((step._graphs.run(m, step._run, args, tag=False).clone(), m.G32.clone(), m._ws["pred"].clone()))
    assert step._graphs.captured() == 1 and not step._graphs.failed
    fail = []
    for i, (l, g, p) in enumerate(outs[1:], 1):
        if not (_bits_equal(l, outs[0][0]) and _bits_equal(g, outs[0][1]) and _bits_equal(p, outs[0][2])):
            fail.append(f"graph replay {i} differs from the eager step")
    keep = outs[0]
    m.set_activation_memory_limit(m.activation_plan.min_bytes)  # only the all-recompute plan fits
    step.use_cuda_graph = False
    r = nf4_check._one_step(m, "qwen", batch, step)
    recomputed = len(m.activation_plan.recompute)
    if not (abs(r[0] - float(keep[0])) == 0 and _bits_equal(r[2], keep[1]) and _bits_equal(r[1], keep[2])):
        fail.append("recompute differs from keep")
    m.set_activation_memory_limit(None)
    # the inference forward has no reductions across CTAs: two forwards agree
    x = torch.cat([batch["noise"], batch["control_latents"]], 1)
    ts = torch.full((2,), 0.5, device="cuda")
    with torch.no_grad():
        f = [m(hidden_states=x, encoder_hidden_states=batch["prompt_embeds"], timestep=ts, img_shapes=batch["img_shapes"])[0].clone()
             for _ in range(2)]
    if not _bits_equal(f[0], f[1]):
        fail.append("inference forwards differ")
    # the gap this closes: two flag-off steps (reported, not asserted)
    torch.use_deterministic_algorithms(False)
    a, b = nf4_check._one_step(m, "qwen", batch, step), nf4_check._one_step(m, "qwen", batch, step)
    off_diff = int((a[2].view(torch.int32) != b[2].view(torch.int32)).sum())
    res = dict(recomputed_blocks=recomputed, flag_off_g32_elements_differing=off_diff, g32_elements=a[2].numel(),
               flag_off_loss_equal=a[0] == b[0], fail=fail, gpu=torch.cuda.get_device_name())
    assert not fail, fail
    return res


def _twin_parity(kind):
    torch = _det()
    import bench
    import fp8_check
    import nf4_check
    mod = fp8_check if kind == "fp8" else nf4_check
    res = {}
    for family, name, over in (("qwen", "qwen_edit", dict(B=1, blocks=3)), ("flux", "flux_kontext", dict(B=1, nd=2, ns=2))):
        cfg = dict(bench.CONFIGS[name], **over)
        batch = nf4_check._fixed(nf4_check.device_batch(cfg, name), family)
        m = mod.build(family, cfg, True)
        r = mod.bf16_twin(m)
        r.add_adapter(cfg["r"], cfg["r"], target_modules=m.peft_config[m.adapter_name].target_modules, b_std=0.02)
        a, b = nf4_check._one_step(m, family, batch), nf4_check._one_step(r, family, batch)
        res[family] = dict(loss_equal=a[0] == b[0], pred_equal=_bits_equal(a[1], b[1]), g32_equal=_bits_equal(a[2], b[2]))
        del m, r
        torch.cuda.empty_cache()
    res["gpu"] = torch.cuda.get_device_name()
    assert all(all(v.values()) for k, v in res.items() if k != "gpu"), res
    return res


def _lora_grad(name):
    def run():
        torch = _det()
        import lora_grad_check as lgc
        from qflux_b200 import lib
        real = lgc.oracle_grads
        calls = {"n": 0}

        def oracle_flag_off(*a, **k):  # torch's eager attention backward has no deterministic kernel; the oracle is not under test
            torch.use_deterministic_algorithms(False)
            try:
                return real(*a, **k)
            finally:
                torch.use_deterministic_algorithms(True)
        lgc.oracle_grads = oracle_flag_off
        real_attn = lib.attn_bwd_det

        def counted(*a, **k):
            calls["n"] += 1
            return real_attn(*a, **k)
        lib.attn_bwd_det = counted
        res = {**lgc.TINY, **lgc.FULL_WIDTH}[name]()
        out = lgc._summary(res)
        out["det_attn_bwd_calls"] = calls["n"]
        assert not res["fail"] and calls["n"] > 0, (res["fail"], calls)
        return out
    return run


CASES = dict(attn_kernels=attn_kernels, reductions=reductions,
             r2r_qwen_ragged_b2=lambda: _three_steps("qwen", "qwen_multires", txt=[352, 200], blocks=4),
             r2r_qwen_edit_plus=lambda: _three_steps("qwen", "qwen_plus_sharded", blocks=4),
             r2r_qwen_multires=lambda: _three_steps("qwen", "qwen_multires", blocks=4),
             r2r_flux_yaml=lambda: _three_steps("flux", "flux_kontext", nd=2, ns=4),
             graph_and_recompute=graph_and_recompute,
             fp8_vs_bf16=lambda: _twin_parity("fp8"), nf4_vs_bf16=lambda: _twin_parity("nf4"))
import lora_grad_check  # noqa: E402

for _n in {**lora_grad_check.TINY, **lora_grad_check.FULL_WIDTH}:
    CASES[f"lora_grad_{_n}"] = _lora_grad(_n)

if __name__ == "__main__":
    harness.main(CASES, os.path.abspath(__file__), "determinism_check.log")
