"""Throughput and peak memory of the fused training step at batch sizes whose saved activations need not fit an 80 GB H100:
the training workspace recomputes the activations of the blocks that do not fit (DESIGN.md §3, `dit.activation_plan`).

    python tools/recompute_bench.py [case ...]       (one subprocess per case via tools/harness.py, which also logs each result line)

Cases: full-depth Qwen-Image-Edit 512² at B = 1, 2, 4, 8; Edit-Plus (target + 2 controls) at B = 1, 2, 4; FLUX-Kontext with the YAML
target set at B = 2, 4, 8; and `library_step_ckpt`, the eager-PyTorch B = 4 step with activation checkpointing (tools/library_bar.py).
Each fused case reports the batch, the recomputed-block count, ms/step from device events after warm-up (eager step, graph capture,
first replay), images/s, peak device memory, the loss, whether the prediction and the LoRA gradient of the last step are finite, and
what the step allocated beyond the planned workspace (the quantity ACTIVATION_HEADROOM must cover), with the GPU name and power limit.
"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "qwen-image-finetune_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import harness  # noqa: E402

STEPS, WARMUP = 5, 3


def _gpu():
    import torch
    try:
        pl = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the number is still valid; say why the power limit is missing
        pl = f"unavailable ({type(e).__name__})"
    return dict(gpu=torch.cuda.get_device_name(), power_limit=pl)


def fused(config, B):
    import torch
    import bench
    from qflux_b200 import mmdit_base
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
    at_plan = {}
    real = mmdit_base.plan_activation_memory

    def recording(blocks, fixed, limit):  # device memory in use when the workspace is planned
        at_plan.update(allocated=torch.cuda.memory_allocated(dev), reserved=torch.cuda.memory_reserved(dev))
        return real(blocks, fixed, limit)
    mmdit_base.plan_activation_memory = recording
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
    ms = e0.elapsed_time(e1) / STEPS
    plan = m.activation_plan
    peak, peak_res = torch.cuda.max_memory_allocated(dev), torch.cuda.max_memory_reserved(dev)
    pred, grad = m._ws["pred"], m.G32
    gib = lambda b: round(b / 2 ** 30, 2)
    return dict(config=config, B=B, blocks=m.L + m.Ls, recomputed_blocks=len(plan.recompute), ms_per_step=round(ms, 1),
                images_per_s=round(B / ms * 1e3, 3), peak_gb=gib(peak), peak_reserved_gb=gib(peak_res), workspace_gb=gib(plan.bytes),
                limit_gb=gib(plan.limit) if plan.limit is not None else None,
                beyond_workspace_gb=gib(peak - at_plan["allocated"] - plan.bytes),
                reserved_beyond_workspace_gb=gib(peak_res - at_plan["reserved"] - plan.bytes),
                loss=float(loss), finite=bool(torch.isfinite(loss).all() and torch.isfinite(pred).all() and torch.isfinite(grad).all()),
                **_gpu())


def library_step_ckpt():
    import library_bar
    return dict(library_bar.step_ckpt(), **_gpu())


CASES = {f"qwen_edit_b{B}": (lambda B=B: fused("qwen_edit", B)) for B in (1, 2, 4, 8)}
CASES.update({f"qwen_plus_b{B}": (lambda B=B: fused("qwen_plus_sharded", B)) for B in (1, 2, 4)})
CASES.update({f"flux_kontext_b{B}": (lambda B=B: fused("flux_kontext", B)) for B in (2, 4, 8)})
CASES["library_step_ckpt"] = library_step_ckpt

if __name__ == "__main__":
    harness.main(CASES, os.path.abspath(__file__), "recompute_bench.log")
