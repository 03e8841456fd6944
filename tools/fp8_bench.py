"""Throughput and peak memory of the fused training step with FP8-resident frozen block weights (a float8-e4m3fn base checkpoint,
`frozen_weights="fp8"`) against the same step with bf16-resident weights, point by point in one run.

    python tools/fp8_bench.py [case ...]       (one subprocess per case via tools/harness.py, which also logs each result line)

Cases: full-depth Qwen-Image-Edit 512² at B = 1, 2, 4, 8; FLUX-Kontext with the YAML target set at B = 2, 4, 8.  In each case the
FP8 step runs first and the bf16 step second in the same process (the FP8 model is freed in between), each with the harness of
tools/nf4_bench.py: ms/step from device events over 5 steps after 3 warm-up steps (eager step, graph capture, first replay),
images/s, peak device memory, recomputed blocks, with the GPU name and power limit.  `expand_qwen_double` times one
qfx_fp8_expand of a full Qwen double block (reads 340 MB, writes 680 MB).  Halving the frozen weights (20.4 GB saved for Qwen,
11.9 GB for FLUX) lets the activation planner keep more blocks; each block fill costs an expansion pass over HBM.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "qwen-image-finetune_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import fp8_check  # noqa: E402
import harness  # noqa: E402
import nf4_check  # noqa: E402
import recompute_bench  # noqa: E402

STEPS, WARMUP = recompute_bench.STEPS, recompute_bench.WARMUP


def _run(config, B, fp8):
    import gc
    import torch
    import bench
    from qflux_b200.optim import FusedLoraAdamW
    torch.manual_seed(1234)
    cfg = dict(bench.CONFIGS[config], B=B)
    family = cfg["model"]
    m = fp8_check.build(family, cfg, fp8=fp8)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    step = nf4_check._step(m, family)
    opt = FusedLoraAdamW(m, lr=1e-4)
    batch = nf4_check.device_batch(cfg, config)
    for _ in range(WARMUP):
        step.train_step(batch, opt)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(STEPS):
        loss = step.train_step(batch, opt)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / STEPS
    res = dict(frozen_weights="fp8" if fp8 else "bf16", recomputed_blocks=len(m.activation_plan.recompute), ms_per_step=round(ms, 1),
               images_per_s=round(B / ms * 1e3, 3), peak_gb=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
               graphs_captured=step._graphs.captured(), loss=float(loss))
    del m, step, opt, batch
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return res


def point(config, B):
    return dict(config=config, B=B, fp8=_run(config, B, True), bf16=_run(config, B, False), **recompute_bench._gpu())


CASES = {f"qwen_edit_b{B}": (lambda B=B: point("qwen_edit", B)) for B in (1, 2, 4, 8)}
CASES.update({f"flux_kontext_b{B}": (lambda B=B: point("flux_kontext", B)) for B in (2, 4, 8)})
CASES["expand_qwen_double"] = fp8_check.kernel_qwen_double

if __name__ == "__main__":
    harness.main(CASES, os.path.abspath(__file__), "fp8_bench.log")
