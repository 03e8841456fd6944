"""Cost of torch.use_deterministic_algorithms(True) on the fused training step, flag off and on alternating in one process:

    python tools/determinism_bench.py [case ...]       (one subprocess per case via tools/harness.py, which logs each result line)

Cases: full-depth Qwen-Image-Edit 512² at B = 1 and B = 4, Edit-Plus (target + 2 controls) at B = 1, FLUX-Kontext with the YAML
target set at B = 2, and `attn_bwd`, the stand-alone attention backward of both kernels at the benchmark shape (B = 4, H = 24,
S = 2400, 40-token prompt).  A step case runs the same model, batch and FusedLoraAdamW through ROUNDS rounds of (flag off, flag on);
each round drops the CUDA graphs and the training workspace, warms up (the workspace is planned and the graph captured again)
and times STEPS steps with device events.  Reported per setting: the median ms/step over the rounds, images/s, and the peak device memory of
its rounds, with the GPU name and power limit read in the same run.
"""
import gc
import os
import sys

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "qwen-image-finetune_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import harness  # noqa: E402
import recompute_bench  # noqa: E402

STEPS, WARMUP, ROUNDS = 5, 3, 2


def step_case(config, B):
    import torch
    import bench
    from qflux_b200.optim import FusedLoraAdamW
    from qflux_b200.train_step import FluxKontextStep, QwenImageEditStep
    dev = torch.device("cuda", 0)
    torch.manual_seed(1234)
    cfg = dict(bench.CONFIGS[config], B=B)
    if cfg["model"] == "qwen":
        m = bench.build_model(dev, cfg["blocks"], cfg)
        step = QwenImageEditStep(m, "mse", max_grad_norm=1.0)
    else:
        m = bench.build_flux(dev, cfg, 1.0)
        step = FluxKontextStep(m, "mse", max_grad_norm=1.0)
    opt = FusedLoraAdamW(m, lr=1e-4)
    host = bench.make_batch(cfg, config, host=False)
    bf_keys = ("image_latents", "control_latents", "prompt_embeds", "pooled_prompt_embeds")
    batch = {k: (v.to(dev, torch.bfloat16) if k in bf_keys else (v.to(dev) if torch.is_tensor(v) else v)) for k, v in host.items()}
    ms, peak, recomputed = {False: [], True: []}, {False: 0, True: 0}, {}
    for _ in range(ROUNDS):
        for det in (False, True):
            torch.use_deterministic_algorithms(det)
            # a captured graph keeps the workspace it was recorded on alive: drop both, so that each setting plans its workspace
            # against the same free memory
            step._graphs.clear()
            m.set_activation_memory_limit(None)
            gc.collect()
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats(dev)
            for _ in range(WARMUP):
                step.train_step(batch, opt)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(STEPS):
                loss = step.train_step(batch, opt)
            e1.record()
            torch.cuda.synchronize()
            assert bool(torch.isfinite(loss).all()) and m._ws["det"] == det
            ms[det].append(e0.elapsed_time(e1) / STEPS)
            peak[det] = max(peak[det], torch.cuda.max_memory_allocated(dev))
            recomputed[det] = len(m.activation_plan.recompute)
    torch.use_deterministic_algorithms(False)
    out = dict(config=config, B=B, blocks=m.L + m.Ls)
    for det, tag in ((False, "off"), (True, "on")):
        med = sorted(ms[det])[len(ms[det]) // 2]
        out[tag] = dict(ms_per_step=round(med, 1), ms_rounds=[round(x, 1) for x in ms[det]], images_per_s=round(B / med * 1e3, 3),
                        peak_gb=round(peak[det] / 2 ** 30, 2), recomputed_blocks=recomputed[det])
    out["cost_pct"] = round(100 * (out["on"]["ms_per_step"] / out["off"]["ms_per_step"] - 1), 1)
    return dict(out, **recompute_bench._gpu())


def attn_bwd():
    """qfx_attn_bwd (atomic dQ, the caller's zero fill included, as the step runs it) vs qfx_attn_bwd_det at the benchmark shape."""
    import torch
    from qflux_b200 import lib
    B, H, S, T = 4, 24, 2400, 352
    g = torch.Generator(device="cuda").manual_seed(0)
    Q, K, V, dO = (torch.randn(B, H, S, 128, device="cuda", generator=g).bfloat16() for _ in range(4))
    txt_len = torch.full((B,), 40, dtype=torch.int32, device="cuda")
    ot, oi = torch.empty(B * T, H * 128, device="cuda", dtype=torch.bfloat16), torch.empty(B * (S - T), H * 128, device="cuda",
                                                                                             dtype=torch.bfloat16)
    lse = torch.empty(B, H, S, device="cuda")
    lib.attn_fwd(Q, K, V, ot, oi, T, lse, txt_len=txt_len)
    delta = torch.randn(B, H, S, device="cuda") * 0.1
    dQ, dK, dV = torch.empty(B, H, S, 128, device="cuda"), torch.empty_like(Q), torch.empty_like(Q)
    res = {}
    for _ in range(ROUNDS):  # alternate the two kernels
        for name, fn in (("atomic", lib.attn_bwd), ("deterministic", lib.attn_bwd_det)):
            def run(fn=fn):
                dQ.zero_()
                fn(Q, K, V, dO, lse, delta, dQ, dK, dV, txt_len=txt_len, split=T)
            res.setdefault(name, []).append(harness.time_cuda(run, iters=20, warmup=3))
    out = {k: round(sorted(v)[len(v) // 2], 3) for k, v in res.items()}
    # the tile products a backward runs (non-causal, dense): atomic 5 (S, dP, dV, dK, dQ), deterministic 7 (S and dP twice)
    return dict(shape=dict(B=B, H=H, S=S, split=T, txt_len=40), ms=out, ratio=round(out["deterministic"] / out["atomic"], 3),
                **recompute_bench._gpu())


CASES = {"qwen_edit_b1": lambda: step_case("qwen_edit", 1), "qwen_edit_b4": lambda: step_case("qwen_edit", 4),
         "qwen_plus_b1": lambda: step_case("qwen_plus_sharded", 1), "flux_kontext_b2": lambda: step_case("flux_kontext", 2),
         "attn_bwd": attn_bwd}

if __name__ == "__main__":
    harness.main(CASES, os.path.abspath(__file__), "determinism_bench.log")
