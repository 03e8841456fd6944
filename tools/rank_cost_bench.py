"""What a wider LoRA rank costs at full depth: bench.py's Qwen-Image-Edit (B = 1, default targets) and FLUX-Kontext (B = 2, the YAML
target set) models at r = 16, 64 and 128, each trained with FusedLoraAdamW (clip 1.0).

    python tools/rank_cost_bench.py [case ...]     (one subprocess per point via tools/harness.py, which also logs each result line)

Per point: WARMUP steps, then STEPS steps timed from device events (best of ROUNDS), images/s, the peak device memory, the blocks
the activation plan recomputes, the LoRA elements and the bytes of the LoRA state (fp32 + bf16 gradient, bf16 parameters, two fp32
AdamW moments: 16 B per element), and the card's name and power limit.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "qwen-image-finetune_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import harness  # noqa: E402
import recompute_bench  # noqa: E402

WARMUP, STEPS, ROUNDS = 3, 5, 2


def point(config, B, r):
    import torch
    import bench
    import nf4_check
    from qflux_b200.optim import FusedLoraAdamW
    from adam8bit_bench import _timed
    dev = torch.device("cuda", 0)
    torch.manual_seed(1234)
    cfg = dict(bench.CONFIGS[config], B=B, r=r)
    family = cfg["model"]
    m = bench.build_model(dev, cfg["blocks"], cfg) if family == "qwen" else bench.build_flux(dev, cfg, 1.0)
    step = nf4_check._step(m, family)
    batch = nf4_check.device_batch(cfg, config)
    torch.cuda.reset_peak_memory_stats()
    opt = FusedLoraAdamW(m, lr=1e-4)
    for _ in range(WARMUP):
        step.train_step(batch, opt)
    ms = min(_timed(lambda: step.train_step(batch, opt), STEPS) for _ in range(ROUNDS))
    n = m.G32.numel()
    return dict(config=config, B=B, r=r, rp=m.lora_rp, ms_per_step=round(ms, 2), images_per_s=round(B / ms * 1e3, 3),
                peak_gb=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2), recomputed_blocks=len(m.activation_plan.recompute),
                lora_elements=n, lora_state_gb=round(16 * n / 1e9, 2), finite=bool(torch.isfinite(m.G32).all()),
                **recompute_bench._gpu())


CASES = {}
for _cfg, _B in (("qwen_edit", 1), ("flux_kontext", 2)):
    for _r in (16, 64, 128):
        CASES[f"{_cfg}_b{_B}_r{_r}"] = (lambda c, B, r: lambda: point(c, B, r))(_cfg, _B, _r)

if __name__ == "__main__":
    harness.main(CASES, os.path.abspath(__file__), "rank_cost_bench.log")
