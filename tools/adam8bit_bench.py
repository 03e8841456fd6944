"""What the configs' 8-bit Adam costs: FusedLoraAdam8bit against FusedLoraAdamW, alternated in one process.

    python tools/adam8bit_bench.py [case ...]     (one subprocess per case via tools/harness.py, which also logs each result line)

  optimizer_flux_yaml  the optimizer call alone (clip norm + update; qfx_fused_adam8bit vs qfx_fused_adamw) on flat buffers laid out like
                       the FLUX-Kontext YAML target set at r = 32 (172 M elements, tools/prodigy_check.py FlatLora), from CUDA events over
                       ITERS launches, best of ROUNDS alternated rounds; the optimizer-state bytes of both, computed from the shapes
                       (8-bit: 2 B per element + 8 B per 256-element block, plus the fp32 path's 8 B per element; AdamW: 8 B per element)
                       and the bytes one call moves (8-bit: 4 B norm read + 4 B gradient + 2 x 2 B codes + 2 x 2 B parameter per
                       element = 16 B; AdamW: 4 + 4 + 2 x 8 + 2 x 2 = 28 B).
  flux_kontext_b2 / qwen_edit_b1
                       full-depth `train_step` time of bench.py's models and batches (FLUX-Kontext YAML targets, r = 32, B = 2;
                       Qwen-Image-Edit, r = 16, B = 1) with each optimizer built after the model's first training step, WARMUP steps then
                       STEPS timed from device events, best of ROUNDS alternated rounds; the optimizer step alone; the peak device memory.
  Every case prints the card's name and power limit.  bitsandbytes' own Adam8bit (after finalize_grads) is timed only when the
  package is importable; otherwise it is reported as not measured.
"""
import gc
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "qwen-image-finetune_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import harness  # noqa: E402
import recompute_bench  # noqa: E402

WARMUP, STEPS, ROUNDS, ITERS = 3, 5, 3, 50
ARGS = dict(lr=1e-4, betas=(0.9, 0.999))  # the configs' init_args


def _timed(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def _bnb():
    try:
        import bitsandbytes  # noqa: F401
        return True
    except ImportError:
        return False


def optimizer_flux_yaml():
    import torch
    from qflux_b200 import lib
    from prodigy_check import FlatLora, _flux_yaml_shapes
    from adam8bit_check import Flat
    fl_p = FlatLora(_flux_yaml_shapes(), 32, 11)
    n = fl_p.n
    fl = Flat(fl_p.members, n, "cuda")
    G = fl_p.grads(0, 5)
    m, v, sumsq = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda"), torch.zeros(1, device="cuda")
    step = {"n": 0}

    def adam8bit():
        step["n"] += 1
        fl.step(G, 1e-4, step["n"])

    def adamw():
        step["n"] += 1
        lib.fused_adamw(fl.tables, G, m, v, sumsq, 1.0, 1.0, 1e-4, 0.9, 0.999, 1e-8, 0.01, step["n"])
    best = {}
    for _ in range(ROUNDS):
        for name, fn in (("fused_adam8bit", adam8bit), ("fused_adamw", adamw)):
            fn()
            ms = _timed(fn, ITERS)
            best[name] = min(best.get(name, ms), ms)
    n8 = int(fl.bw.sum())
    nblocks = sum(-(-p.numel() // 256) for p, _ in fl_p.members if p.numel() >= 4096)
    state8 = 2 * n8 + 8 * nblocks + 8 * (n - n8)
    res = dict(elements=n, elements_fp32_path=n - n8,
               ms=dict((k, round(v, 3)) for k, v in best.items()),
               state_gb=dict(fused_adam8bit=round(state8 / 1e9, 3), fused_adamw=round(8 * n / 1e9, 3)),
               bytes_per_element=dict(fused_adam8bit=16, fused_adamw=28),
               achieved_tb_s=dict(fused_adam8bit=round(16 * n / best["fused_adam8bit"] / 1e9, 2),
                                  fused_adamw=round(28 * n / best["fused_adamw"] / 1e9, 2)),
               bitsandbytes="not measured (bitsandbytes is not installed)" if not _bnb() else "see the step cases",
               **recompute_bench._gpu())
    return res


def _make(setting, m):
    from qflux_b200.optim import FusedLoraAdam8bit, FusedLoraAdamW
    if setting == "fused_adam8bit":
        return FusedLoraAdam8bit(m, **ARGS, max_grad_norm=1.0)
    if setting == "fused_adamw":
        return FusedLoraAdamW(m, **ARGS)
    import bitsandbytes as bnb
    return bnb.optim.Adam8bit(list(m.parameters()), **ARGS)


def point(config, B):
    import torch
    import bench
    import nf4_check
    from qflux_b200.optim import FusedLoraOptimizer
    dev = torch.device("cuda", 0)
    torch.manual_seed(1234)
    cfg = dict(bench.CONFIGS[config], B=B)
    family = cfg["model"]
    m = bench.build_model(dev, cfg["blocks"], cfg) if family == "qwen" else bench.build_flux(dev, cfg, 1.0)
    step = nf4_check._step(m, family)
    batch = nf4_check.device_batch(cfg, config)
    step.train_step(batch, None)  # plans and allocates the training workspace before any optimizer state exists
    settings = ["fused_adam8bit", "fused_adamw"] + (["bitsandbytes_adam8bit"] if _bnb() else [])
    best = {}
    torch.cuda.reset_peak_memory_stats()
    for _ in range(ROUNDS):
        for s in settings:
            opt = _make(s, m)
            for _ in range(WARMUP):
                step.train_step(batch, opt)
            ms = _timed(lambda: step.train_step(batch, opt), STEPS)
            fused = isinstance(opt, FusedLoraOptimizer)
            opt_ms = _timed(opt.step if fused else (lambda: (m.finalize_grads(1, 1.0), opt.step())), STEPS)
            tensors = vars(opt).values() if fused else [t for st in opt.state.values() for t in st.values()]
            state = sum(t.numel() * t.element_size() for t in tensors if torch.is_tensor(t) and t.numel() > 1000)
            r = dict(ms_per_step=round(ms, 2), images_per_s=round(B / ms * 1e3, 3), optimizer_step_ms=round(opt_ms, 3),
                     state_gb=round(state / 1e9, 3))
            if s not in best or r["ms_per_step"] < best[s]["ms_per_step"]:
                best[s] = r
            del opt
            gc.collect()
            torch.cuda.empty_cache()
    if not _bnb():
        best["bitsandbytes_adam8bit"] = "not measured (bitsandbytes is not installed)"
    return dict(config=config, B=B, lora_elements=m.G32.numel(), recomputed_blocks=len(m.activation_plan.recompute),
                peak_gb=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2), settings=best, **recompute_bench._gpu())


CASES = dict(optimizer_flux_yaml=optimizer_flux_yaml, flux_kontext_b2=lambda: point("flux_kontext", 2),
             qwen_edit_b1=lambda: point("qwen_edit", 1))

if __name__ == "__main__":
    harness.main(CASES, os.path.abspath(__file__), "adam8bit_bench.log")
