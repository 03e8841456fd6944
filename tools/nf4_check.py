"""GPU checks of NF4-resident frozen weights (4-bit base checkpoints, qflux_b200/nf4.py), one subprocess per case:

    python tools/nf4_check.py [case ...]

  kernel_qwen_double / kernel_flux_single  qfx_nf4_dequant of one full-size block (every NF4 matrix of it in one launch) equals the
                                           restated rule (torch fp32 product, bf16 rounding) bit for bit
  qwen_full_parity                         full-depth Qwen-Image-Edit, B = 1: the NF4 model and a bf16 model holding the dequantized
                                           weights give the same prediction and loss, and LoRA gradients that differ by no more than
                                           two runs of the bf16 model differ; the NF4 step's peak memory is below the bf16 step's by at
                                           least 90 % of the computed saving
  graph_replay                             a CUDA-graph replayed NF4 training step equals its eager run (Qwen and FLUX)
  infer_replay                             the replayed NF4 inference forward is bit-exact and the graph cache captured
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "qwen-image-finetune_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import harness  # noqa: E402


def fill_nf4_model(m, seed=1234):
    """Random NF4 codes with absmax in [0.02, 0.04) (weights of std ~0.017, like N(0, 0.02^2)); the bf16 tensors as bench.py's
    initialisation: N(0, 0.02^2) matrices, zero biases, unit q/k norm weights."""
    import torch
    g = torch.Generator(device=m.dev).manual_seed(seed)
    for codes, absmax in m._nf4_store.values():
        codes.copy_(torch.randint(0, 256, codes.shape, device=m.dev, generator=g, dtype=torch.int32).to(torch.uint8))
        absmax.uniform_(0.02, 0.04, generator=g)
    for k, t in m.w.items():
        if torch.is_tensor(t) and (k.endswith("_w") and t.ndim >= 2 and "norm" not in k or k == "norm_out_w"):
            t.normal_(0.0, 0.02, generator=g)
    return m


def bf16_twin(m):
    """A bf16-resident model of m's config holding m's weights, the NF4 matrices dequantized layer by layer with the kernel."""
    import torch
    from qflux_b200 import lib
    r = type(m)(m.config, device=m.dev)
    for k, t in m.w.items():
        if k in m._nf4_store:
            codes, absmax = m._nf4_store[k]
            for l in range(codes.shape[0]):
                lib.nf4_dequant([(codes[l].reshape(-1), absmax[l], r.w[k][l].view(-1), m.nf4_blocksize)])
        else:
            r.w[k].copy_(t)
    torch.cuda.synchronize()
    return r


def build(family, cfg, nf4=True):
    """The bench.py model of `family` (full depth) with NF4-resident or bf16 frozen block weights, with the bench adapter."""
    import torch
    import bench
    from qflux_b200.flux_model import FLUX_KONTEXT_YAML_TARGETS, FluxB200, FluxB200Config
    from qflux_b200.qwen_model import QwenB200Config, QwenImageB200
    dev = torch.device("cuda", 0)
    fw = "nf4" if nf4 else "bf16"
    if family == "qwen":
        m = QwenImageB200(QwenB200Config(num_layers=cfg["blocks"], num_attention_heads=bench.CFG["heads"],
                                         joint_attention_dim=bench.CFG["joint"]), device=dev, frozen_weights=fw)
        targets = None
    else:
        m = FluxB200(FluxB200Config(num_layers=cfg.get("nd", 19), num_single_layers=cfg.get("ns", 38), guidance_embeds=True), device=dev,
                     frozen_weights=fw)
        targets = FLUX_KONTEXT_YAML_TARGETS
    if nf4:
        fill_nf4_model(m)
    else:
        bench._init_weights(m, dev)
    m.add_adapter(cfg["r"], cfg["r"], target_modules=targets, b_std=0.02)
    return m


def device_batch(cfg, name):
    import torch
    import bench
    dev = torch.device("cuda", 0)
    host = bench.make_batch(cfg, name, host=False)
    bf = ("image_latents", "control_latents", "prompt_embeds", "pooled_prompt_embeds")
    return {k: (v.to(dev, torch.bfloat16) if k in bf else (v.to(dev) if torch.is_tensor(v) else v)) for k, v in host.items()}


def _step(m, family):
    from qflux_b200.train_step import FluxKontextStep, QwenImageEditStep
    return (QwenImageEditStep if family == "qwen" else FluxKontextStep)(m, "mse", max_grad_norm=1.0)


def _one_step(m, family, batch, step=None):
    """loss, prediction and flat LoRA gradient of one eager fused step on fixed noise / timestep."""
    step = step or _step(m, family)
    loss = step._run(*step._prepare(batch, batch.get("noise"), batch.get("u") if family == "qwen" else batch.get("timestep")))
    return float(loss), m._ws["pred"].clone(), m.G32.clone()


def _fixed(batch, family):
    import torch
    g = torch.Generator(device="cuda").manual_seed(7)
    b = dict(batch)
    B = b["image_latents"].shape[0]
    b["noise"] = torch.randn(b["image_latents"].shape, device="cuda", generator=g).bfloat16()
    if family == "qwen":
        b["u"] = torch.tensor([0.375] * B)
    else:
        b["timestep"] = torch.full((B,), 0.375, device="cuda", dtype=torch.bfloat16)
    return b


# ------------------------------------------------------------------------------------------------------------------------ cases
def _kernel(kinds):
    import torch
    from qflux_b200 import lib, nf4
    D, bs = 3072, 64
    g = torch.Generator(device="cuda").manual_seed(3)
    segs, refs = [], []
    for n_rows, n_cols in kinds:
        n = n_rows * n_cols
        codes = torch.randint(0, 256, (n // 2,), device="cuda", generator=g, dtype=torch.int32).to(torch.uint8)
        absmax = torch.rand(n // bs, device="cuda", generator=g) * 0.1
        absmax[:7] = torch.tensor([0.0, 1e-40, 3e-39, 1e-38, 65504.0, 1e30, 2.0 ** -126], device="cuda")  # zero, subnormal, huge
        out = torch.empty(n, device="cuda", dtype=torch.bfloat16)
        segs.append((codes, absmax, out, bs))
        idx = torch.stack((codes >> 4, codes & 15), -1).reshape(-1).long()
        refs.append((nf4.NF4_TABLE.cuda()[idx] * absmax.repeat_interleave(bs)).to(torch.bfloat16))
    lib.nf4_dequant(segs)
    ms = harness.time_cuda(lambda: lib.nf4_dequant(segs), iters=20)
    torch.cuda.synchronize()
    mismatch = sum(int((s[2].view(torch.int16) != r.view(torch.int16)).sum()) for s, r in zip(segs, refs))
    nbytes = sum(s[0].numel() + s[1].numel() * 4 + s[2].numel() * 2 for s in segs)
    assert mismatch == 0, mismatch
    return dict(mismatched_elements=mismatch, elements=sum(s[2].numel() for s in segs), ms=round(ms, 3),
                gb_per_s=round(nbytes / ms / 1e6, 1), gpu=torch.cuda.get_device_name(), D=D)


def kernel_qwen_double():
    D = 3072
    return _kernel([(2 * 6 * D, D), (2 * 3 * D, D), (2 * D, D), (2 * 4 * D, D), (2 * D, 4 * D)])


def kernel_flux_single():
    D = 3072
    return _kernel([(3 * D, D), (3 * D, D), (4 * D, D), (D, 5 * D)])


def _rel(a, b):
    return harness.rel_l2(a, b)


def qwen_full_parity():
    import gc
    import torch
    import bench
    cfg = dict(bench.CONFIGS["qwen_edit"], B=1)
    batch = _fixed(device_batch(cfg, "qwen_edit"), "qwen")
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    m = build("qwen", cfg, nf4=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()  # the step's peak (the model's weights are allocated), not the initialisation's temporaries
    a = _one_step(m, "qwen", batch)
    torch.cuda.synchronize()
    peak_nf4 = torch.cuda.max_memory_allocated() - base
    D, L = m.D, m.L
    bf16_bytes = sum(c.numel() * 2 * 2 for c, _ in m._nf4_store.values())
    nf4_bytes = sum(c.numel() + x.numel() * 4 for c, x in m._nf4_store.values()) + sum(r.gbuf.numel() * 2 for r in m._nf4_rings if r is not None)
    r = bf16_twin(m)
    r.add_adapter(cfg["r"], cfg["r"], b_std=0.02)  # the same seeded factors as m's
    del m
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()  # after m is freed: the bf16 step's peak with r's weights allocated
    b = _one_step(r, "qwen", batch)
    c = _one_step(r, "qwen", batch)
    torch.cuda.synchronize()
    peak_bf16 = torch.cuda.max_memory_allocated() - base
    saving = bf16_bytes - nf4_bytes
    res = dict(loss_nf4=a[0], loss_bf16=b[0], loss_bf16_again=c[0], pred_identical=bool(torch.equal(a[1], b[1])),
               grad_rel_nf4_vs_bf16=_rel(a[2], b[2]), grad_rel_bf16_vs_bf16=_rel(c[2], b[2]), peak_nf4_gb=round(peak_nf4 / 2 ** 30, 2),
               peak_bf16_gb=round(peak_bf16 / 2 ** 30, 2), computed_saving_gb=round(saving / 2 ** 30, 2),
               measured_saving_gb=round((peak_bf16 - peak_nf4) / 2 ** 30, 2), recomputed_blocks=len(r.activation_plan.recompute),
               gpu=torch.cuda.get_device_name())
    print(res)
    assert res["pred_identical"] and abs(a[0] - b[0]) <= 1e-6 * abs(b[0])
    assert res["grad_rel_nf4_vs_bf16"] <= 1.5 * res["grad_rel_bf16_vs_bf16"] + 1e-6
    assert peak_bf16 - peak_nf4 >= 0.9 * saving
    return res


def graph_replay():
    import torch
    import bench
    out = {}
    for family, name, cfg in (("qwen", "qwen_edit", dict(bench.CONFIGS["qwen_edit"], B=1, blocks=6)),
                              ("flux", "flux_kontext", dict(bench.CONFIGS["flux_kontext"], B=1, nd=3, ns=3))):
        m = build(family, cfg)
        batch = _fixed(device_batch(cfg, name), family)
        step = _step(m, family)
        args = step._prepare(batch, batch["noise"], batch["u"] if family == "qwen" else batch["timestep"])
        outs = []
        for _ in range(3):  # eager, capture + first replay, replay
            outs.append((float(step._graphs.run(m, step._run, args, tag=False)), m._ws["pred"].clone(), m.G32.clone()))
        assert step._graphs.captured() == 1 and not step._graphs.failed
        for loss, pred, g in outs[1:]:
            assert abs(loss - outs[0][0]) <= 1e-6 * abs(outs[0][0]) and torch.equal(pred, outs[0][1]), family
        out[family] = dict(loss=outs[0][0], grad_rel=max(_rel(g, outs[0][2]) for _, _, g in outs[1:]))
        assert out[family]["grad_rel"] < 1e-2
        del m, step
    return out


def infer_replay():
    import torch
    import bench
    cfg = dict(bench.CONFIGS["qwen_edit"], B=1, blocks=6)
    m = build("qwen", cfg)
    b = _fixed(device_batch(cfg, "qwen_edit"), "qwen")
    x = torch.cat([b["noise"], b["control_latents"]], 1)
    ts = torch.full((1,), 0.5, device="cuda")
    outs = []
    with torch.no_grad():
        for _ in range(4):  # eager (warm), capture + replay, replay, replay
            outs.append(m(hidden_states=x, encoder_hidden_states=b["prompt_embeds"], timestep=ts, img_shapes=b["img_shapes"])[0].clone())
    assert m._infer_graphs.captured() == 1 and not m._infer_graphs.failed
    same = all(torch.equal(o, outs[0]) for o in outs[1:])
    assert same
    return dict(captured=m._infer_graphs.captured(), bit_exact=same)


CASES = dict(kernel_qwen_double=kernel_qwen_double, kernel_flux_single=kernel_flux_single, qwen_full_parity=qwen_full_parity,
             graph_replay=graph_replay, infer_replay=infer_replay)

if __name__ == "__main__":
    if len(sys.argv) == 2 and sys.argv[1] in CASES:  # one case in this process (tests/test_nf4_weights.py)
        print(CASES[sys.argv[1]]())
    else:
        harness.main(CASES, os.path.abspath(__file__), "nf4_check.log")
