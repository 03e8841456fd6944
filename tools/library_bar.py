"""GPU library bar (BASELINE.md §2): what the reference would actually run on one H100 — the eager-PyTorch restatement of its step
(cuBLASLt bf16 GEMMs + F.scaled_dot_product_attention, autograd backward, torch AdamW on the LoRA parameters) — and the library
attention kernels (cuDNN / flash SDPA, forward and backward) at the benchmark shape, timed beside our own kernels.

    python tools/library_bar.py [attn] [step_ckpt] [step_nockpt]        (run under gpurun; writes gpurun_out/library_bar.json)

The oracle is used here as a BASELINE being measured (like bench.py's cpu_baseline leg), never as part of the product path.
"""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "qwen-image-finetune_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

BF = torch.bfloat16


def _time(fn, iters=10, warmup=3, flush=None):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def attn_library(B=4, H=24, S=2400, d=128):
    """cuDNN / flash / mem-efficient SDPA forward and backward at the Qwen-Image-Edit shape, beside qfx_attn_fwd / qfx_attn_bwd."""
    from torch.nn.attention import SDPBackend, sdpa_kernel
    from qflux_b200 import lib
    g = torch.Generator(device="cuda").manual_seed(0)
    Q, K, V = ((torch.randn(B, H, S, d, device="cuda", generator=g)).to(BF) for _ in range(3))
    dO = torch.randn(B, H, S, d, device="cuda", generator=g).to(BF)
    flush = torch.empty(256 << 20, device="cuda", dtype=torch.uint8)
    f_fwd, f_bwd = 4.0 * B * H * S * S * d, 10.0 * B * H * S * S * d
    out = {}
    for name, be in (("cudnn", SDPBackend.CUDNN_ATTENTION), ("flash", SDPBackend.FLASH_ATTENTION), ("efficient", SDPBackend.EFFICIENT_ATTENTION)):
        try:
            with sdpa_kernel([be]):
                q, k, v = (t.clone().requires_grad_(True) for t in (Q, K, V))
                ms_f = _time(lambda: F.scaled_dot_product_attention(q, k, v), flush=flush)
                o = F.scaled_dot_product_attention(q, k, v)

                def bwd():
                    torch.autograd.grad(o, (q, k, v), dO, retain_graph=True)
                ms_b = _time(bwd, flush=flush)
            out[name] = dict(fwd_ms=round(ms_f, 4), fwd_tflops=round(f_fwd / ms_f / 1e9, 1), bwd_ms=round(ms_b, 4),
                             bwd_tflops=round(f_bwd / ms_b / 1e9, 1))
        except Exception as e:  # backend not available for this shape / build
            out[name] = dict(error=str(e)[:200])
    # ours (same tensors; forward writes token-major output, backward = delta + main kernel, both counted)
    T = 352
    ot, oi = torch.empty(B * T, H * d, device="cuda", dtype=BF), torch.empty(B * (S - T), H * d, device="cuda", dtype=BF)
    lse = torch.empty(B, H, S, device="cuda")
    ms_f = _time(lambda: lib.attn_fwd(Q, K, V, ot, oi, T, lse), flush=flush)
    dot, doi = torch.randn_like(ot), torch.randn_like(oi)
    delta, dOj = torch.empty(B, H, S, device="cuda"), torch.empty(B, H, S, d, device="cuda", dtype=BF)
    dQ, dK, dV = torch.zeros(B, H, S, d, device="cuda"), torch.empty_like(K), torch.empty_like(V)

    def ours_bwd_core():
        dQ.zero_()
        lib.attn_bwd(Q, K, V, dOj, lse, delta, dQ, dK, dV, split=T)

    def ours_bwd_all():
        lib.attn_delta(ot, dot, delta, T, 0, dOj)
        lib.attn_delta(oi, doi, delta, S - T, T, dOj)
        ours_bwd_core()
    ours_bwd_all()
    ms_b = _time(ours_bwd_core, flush=flush)
    ms_ba = _time(ours_bwd_all, flush=flush)
    out["qfx"] = dict(fwd_ms=round(ms_f, 4), fwd_tflops=round(f_fwd / ms_f / 1e9, 1), bwd_ms=round(ms_b, 4),
                      bwd_tflops=round(f_bwd / ms_b / 1e9, 1), bwd_with_delta_and_dq_zero_ms=round(ms_ba, 4))
    return out


def _eager_step(layers, B, ckpt, steps=3, warmup=2, T=352, imgs=((1, 32, 32), (1, 32, 32))):
    """One eager training step of the oracle model in bf16 on the GPU: fwd + flow-matching loss + autograd bwd + clip + AdamW."""
    from oracle import mmdit_oracle as mo
    from torch.utils.checkpoint import checkpoint
    torch.manual_seed(0)
    with torch.device("cuda"):
        m = mo.QwenImageOracle(mo.QwenConfig(num_layers=layers))
    m = m.to(BF)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith("bias"):
                p.zero_()
            elif p.ndim == 1:
                p.fill_(1.0)
            else:
                p.normal_(0, 0.02)
    mo.add_lora_adapter(m, r=16, alpha=16, b_std=0.02)
    m = m.to("cuda", BF)
    if ckpt:  # the reference's `gradient_checkpointing: true` (transformer_qwenimage.py:640-652): one checkpoint per block
        for blk in m.transformer_blocks:
            fwd = blk.forward
            blk.forward = (lambda f: (lambda *a, **k: checkpoint(f, *a, use_reentrant=False, **k)))(fwd)
    params = [p for p in m.parameters() if p.requires_grad]
    opt = torch.optim.AdamW(params, lr=1e-4)
    imgs = [tuple(s) for s in imgs]
    L, Lc = imgs[0][1] * imgs[0][2], sum(f * h * w for f, h, w in imgs[1:])
    g = torch.Generator(device="cuda").manual_seed(1)
    x = dict(image_latents=torch.randn(B, L, 64, device="cuda", generator=g).to(BF), control_latents=torch.randn(B, Lc, 64, device="cuda", generator=g).to(BF),
             prompt_embeds=(torch.randn(B, T, 3584, device="cuda", generator=g) * 3).to(BF),
             prompt_embeds_mask=torch.ones(B, T, dtype=torch.int64, device="cuda"), img_shapes=[list(imgs)] * B)

    def step():
        noise = torch.randn(B, L, 64, device="cuda", dtype=BF)
        loss, _ = mo.qwen_compute_loss(m, **x, noise=noise, u=torch.rand(B))
        loss.backward()
        torch.nn.utils.clip_grad_norm_(params, 1.0)
        opt.step()
        opt.zero_grad(set_to_none=True)
        return loss
    torch.cuda.reset_peak_memory_stats()
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    for _ in range(steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    wall = (time.perf_counter() - t0) / steps * 1e3
    r = dict(layers=layers, B=B, checkpointing=ckpt, ms_per_step=round(ms, 2), wall_ms_per_step=round(wall, 2), images_per_s=round(B / ms * 1e3, 3),
             peak_mem_gb=round(torch.cuda.max_memory_allocated() / 2 ** 30, 1), loss=float(loss))
    del m, opt, params
    torch.cuda.empty_cache()
    return r


def step_ckpt():
    """Full depth (60 blocks), B=4, gradient checkpointing on — the reference's shipped configuration (configs/*.yaml)."""
    return _eager_step(60, 4, True)


def step_nockpt():
    """Without checkpointing the eager activations of 60 blocks at B=4 do not fit one GPU: measure the deepest model that fits and
    scale linearly in depth (the embed / head share is < 1 %)."""
    for layers in (60, 40, 28, 20, 12):
        try:
            r = _eager_step(layers, 4, False)
            r["images_per_s_at_60_blocks"] = round(r["images_per_s"] * layers / 60, 3)
            r["ms_per_step_at_60_blocks"] = round(r["ms_per_step"] * 60 / layers, 1)
            return r
        except torch.OutOfMemoryError:
            torch.cuda.empty_cache()
    return dict(error="out of memory at every depth tried")


CASES = {"attn": attn_library, "step_ckpt": step_ckpt, "step_nockpt": step_nockpt}

if __name__ == "__main__":
    only = sys.argv[1:] or list(CASES)
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    path = os.path.join(ROOT, "gpurun_out", "library_bar.json")
    res = json.load(open(path)) if os.path.exists(path) else {}
    for name in only:
        try:
            res[name] = CASES[name]()
        except Exception as e:
            res[name] = dict(error=repr(e)[:300])
        print(name, json.dumps(res[name]), flush=True)
        json.dump(res, open(path, "w"), indent=1)
