"""GPU checks of FP8-resident frozen weights (float8-e4m3fn base checkpoints, qflux_b200/fp8.py), one subprocess per case:

    python tools/fp8_check.py [case ...]

  kernel_all_codes                         qfx_fp8_expand of all 256 codes, in eight segments of different lengths, equals torch's
                                           `.to(torch.bfloat16)` bit for bit (the two NaN codes: NaN on both sides)
  kernel_qwen_double / kernel_flux_single  qfx_fp8_expand of one full-size block (every FP8 matrix of it in one launch) equals torch's
                                           conversion bit for bit; time and bytes/s of the launch
  qwen_step_parity / flux_step_parity      a multi-block full-width training step (Qwen 6 blocks; FLUX 3 double + 3 single, YAML
                                           targets): the FP8 model and a bf16 model holding the upcast weights give the same
                                           prediction bit for bit; the loss and the whole LoRA gradient are no further apart than
                                           two runs of the same model are (the loss and some gradient sums are reduced with atomics);
                                           under torch.use_deterministic_algorithms(True) the loss and every LoRA gradient tensor
                                           agree bit for bit
  graph_replay                             a CUDA-graph replayed FP8 training step equals its eager run (Qwen and FLUX)
  infer_replay                             the replayed FP8 inference forward is bit-exact and the graph cache captured
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "qwen-image-finetune_b200"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import harness  # noqa: E402
import nf4_check  # noqa: E402  (device batches and the one-step recipe are shared)
import recompute_bench  # noqa: E402


def fill_fp8_model(m, seed=1234):
    """e4m3fn codes of N(0, 0.02^2) weights (subnormals included), layer by layer; the bf16 tensors as bench.py's initialisation."""
    import torch
    g = torch.Generator(device=m.dev).manual_seed(seed)
    for codes in m._fp8_store.values():
        for l in range(codes.shape[0]):
            x = torch.randn(codes.shape[1:], device=m.dev, generator=g) * 0.02
            codes[l].view(torch.uint8).copy_(x.to(torch.float8_e4m3fn).view(torch.uint8))
    for k, t in m.w.items():
        if torch.is_tensor(t) and (k.endswith("_w") and t.ndim >= 2 and "norm" not in k or k == "norm_out_w"):
            t.normal_(0.0, 0.02, generator=g)
    return m


def bf16_twin(m):
    """A bf16-resident model of m's config holding m's weights, the FP8 matrices upcast by torch (not by the kernel)."""
    import torch
    r = type(m)(m.config, device=m.dev)
    for k, t in m.w.items():
        if k in m._fp8_store:
            for l, c in enumerate(m._fp8_store[k]):
                r.w[k][l].copy_(c.to(torch.bfloat16))
        else:
            r.w[k].copy_(t)
    torch.cuda.synchronize()
    return r


def build(family, cfg, fp8=True):
    """The bench.py model of `family` with FP8-resident or bf16 frozen block weights, with the bench adapter."""
    import torch
    import bench
    from qflux_b200.flux_model import FLUX_KONTEXT_YAML_TARGETS, FluxB200, FluxB200Config
    from qflux_b200.qwen_model import QwenB200Config, QwenImageB200
    dev = torch.device("cuda", 0)
    fw = "fp8" if fp8 else "bf16"
    if family == "qwen":
        m = QwenImageB200(QwenB200Config(num_layers=cfg["blocks"], num_attention_heads=bench.CFG["heads"],
                                         joint_attention_dim=bench.CFG["joint"]), device=dev, frozen_weights=fw)
        targets = None
    else:
        m = FluxB200(FluxB200Config(num_layers=cfg.get("nd", 19), num_single_layers=cfg.get("ns", 38), guidance_embeds=True), device=dev,
                     frozen_weights=fw)
        targets = FLUX_KONTEXT_YAML_TARGETS
    if fp8:
        fill_fp8_model(m)
    else:
        bench._init_weights(m, dev)
    m.add_adapter(cfg["r"], cfg["r"], target_modules=targets, b_std=0.02)
    return m


# ------------------------------------------------------------------------------------------------------------------------ cases
def _check(segs):
    import torch
    bad = 0
    for codes, out in segs:
        ref = codes.view(torch.float8_e4m3fn).to(torch.bfloat16)
        nan = ref.isnan()
        bad += int(((out.view(torch.int16) != ref.view(torch.int16)) & ~nan).sum()) + int((out.isnan() != nan).sum())
    return bad


def kernel_all_codes():
    import torch
    from qflux_b200 import lib
    segs = []
    for i, n in enumerate((16, 256, 272, 4096, 4112, 48, 65536, 1024)):
        codes = (torch.arange(n, device="cuda", dtype=torch.int32) * (i + 1) % 256).to(torch.uint8)
        segs.append((codes, torch.full((n,), float("nan"), device="cuda", dtype=torch.bfloat16)))
    lib.fp8_expand(segs)
    torch.cuda.synchronize()
    covered = torch.unique(torch.cat([c for c, _ in segs])).numel()
    bad = _check(segs)
    assert covered == 256 and bad == 0, (covered, bad)
    # the values that matter most: -0, the subnormals and the extremes
    c = torch.tensor([0x80, 0x01, 0x02, 0x07, 0x08, 0x7E, 0xFE, 0x00, 0x81, 0x87] + [0] * 6, device="cuda", dtype=torch.uint8)
    o = torch.empty(16, device="cuda", dtype=torch.bfloat16)
    lib.fp8_expand([(c, o)])
    vals = o.float().tolist()[:10]
    assert o.view(torch.int16)[0].item() == -32768 and vals[1] == 2.0 ** -9 and vals[3] == 7 * 2.0 ** -9 and vals[4] == 2.0 ** -6
    assert vals[5] == 448.0 and vals[6] == -448.0 and vals[8] == -(2.0 ** -9)
    return dict(codes_covered=covered, mismatched_elements=bad, specials=vals, gpu=torch.cuda.get_device_name())


def _kernel(kinds):
    import torch
    from qflux_b200 import lib
    g = torch.Generator(device="cuda").manual_seed(3)
    segs = []
    for n_rows, n_cols in kinds:
        codes = torch.randint(0, 256, (n_rows * n_cols,), device="cuda", generator=g, dtype=torch.int32).to(torch.uint8)
        codes[(codes & 0x7F) == 0x7F] = 0  # finite weights only: an FP8 checkpoint's NaN codes are refused at load
        segs.append((codes, torch.empty(n_rows * n_cols, device="cuda", dtype=torch.bfloat16)))
    lib.fp8_expand(segs)
    torch.cuda.synchronize()
    bad = _check(segs)
    ms = harness.time_cuda(lambda: lib.fp8_expand(segs), iters=20)
    read, written = sum(c.numel() for c, _ in segs), sum(o.numel() * 2 for _, o in segs)
    assert bad == 0, bad
    return dict(mismatched_elements=bad, elements=read, read_mb=round(read / 1e6, 1), written_mb=round(written / 1e6, 1), ms=round(ms, 3),
                gb_per_s=round((read + written) / ms / 1e6, 1), **recompute_bench._gpu())


def kernel_qwen_double():
    D = 3072
    return _kernel([(2 * 6 * D, D), (2 * 3 * D, D), (2 * D, D), (2 * 4 * D, D), (2 * D, 4 * D)])


def kernel_flux_single():
    D = 3072
    return _kernel([(3 * D, D), (3 * D, D), (4 * D, D), (D, 5 * D)])


def _step_parity(family, name, cfg):
    import torch
    import bench
    cfg = dict(bench.CONFIGS[name], **cfg)
    batch = nf4_check._fixed(nf4_check.device_batch(cfg, name), family)
    m = build(family, cfg, fp8=True)
    r = bf16_twin(m)
    r.add_adapter(cfg["r"], cfg["r"], target_modules=m.peft_config[m.adapter_name].target_modules, b_std=0.02)  # same seeded factors
    assert all(torch.equal(p, r._lora_params[k]) for k, p in m._lora_params.items())
    # flag off (the default path): the forward is bit-identical; the loss and some gradient sums end in floating-point atomics, so
    # two runs of one model differ, and the pooled FP8-vs-bf16 distance is held to that rerun spread
    a, a2 = nf4_check._one_step(m, family, batch), nf4_check._one_step(m, family, batch)
    b, b2 = nf4_check._one_step(r, family, batch), nf4_check._one_step(r, family, batch)
    pooled, pooled_noise = harness.rel_l2(a[2], b[2]), max(harness.rel_l2(b2[2], b[2]), harness.rel_l2(a2[2], a[2]))
    # flag on: every reduction in a fixed order, so the two models must agree bit for bit, loss and every LoRA gradient tensor
    torch.use_deterministic_algorithms(True)
    try:
        da, db = nf4_check._one_step(m, family, batch), nf4_check._one_step(r, family, batch)
    finally:
        torch.use_deterministic_algorithms(False)
    va, vb = m.lora_grad_views(da[2]), r.lora_grad_views(db[2])
    differ = [k for k in vb if not torch.equal(va[k].view(torch.int32), vb[k].view(torch.int32))]
    res = dict(family=family, blocks=m.L + m.Ls, pred_identical=bool(torch.equal(a[1], b[1])), loss_fp8=a[0], loss_bf16=b[0],
               loss_bf16_again=b2[0], lora_tensors=len(vb), bf16_rerun_bitwise=bool(torch.equal(b[2], b2[2])),
               grad_rel_fp8_vs_bf16=pooled, grad_rel_rerun=pooled_noise,
               det_pred_identical=bool(torch.equal(da[1], db[1])), det_loss_identical=da[0] == db[0],
               det_differing_tensors=differ[:5], gpu=torch.cuda.get_device_name())
    print(res)
    assert res["pred_identical"] and abs(a[0] - b[0]) <= 1e-6 * abs(b[0]) and pooled <= 2 * pooled_noise + 1e-6
    assert res["det_pred_identical"] and res["det_loss_identical"] and not differ
    return res


def qwen_step_parity():
    return _step_parity("qwen", "qwen_edit", dict(B=1, blocks=6))


def flux_step_parity():
    return _step_parity("flux", "flux_kontext", dict(B=1, nd=3, ns=3))


def graph_replay():
    import torch
    import bench
    out = {}
    for family, name, cfg in (("qwen", "qwen_edit", dict(bench.CONFIGS["qwen_edit"], B=1, blocks=6)),
                              ("flux", "flux_kontext", dict(bench.CONFIGS["flux_kontext"], B=1, nd=3, ns=3))):
        m = build(family, cfg)
        batch = nf4_check._fixed(nf4_check.device_batch(cfg, name), family)
        step = nf4_check._step(m, family)
        args = step._prepare(batch, batch["noise"], batch["u"] if family == "qwen" else batch["timestep"])
        outs = []
        for _ in range(3):  # eager, capture + first replay, replay
            outs.append((float(step._graphs.run(m, step._run, args, tag=False)), m._ws["pred"].clone(), m.G32.clone()))
        assert step._graphs.captured() == 1 and not step._graphs.failed
        for loss, pred, g in outs[1:]:
            assert abs(loss - outs[0][0]) <= 1e-6 * abs(outs[0][0]) and torch.equal(pred, outs[0][1]), family
        out[family] = dict(loss=outs[0][0], grad_rel=max(harness.rel_l2(g, outs[0][2]) for _, _, g in outs[1:]))
        assert out[family]["grad_rel"] < 1e-2
        del m, step
    return out


def infer_replay():
    import torch
    import bench
    cfg = dict(bench.CONFIGS["qwen_edit"], B=1, blocks=6)
    m = build("qwen", cfg)
    b = nf4_check._fixed(nf4_check.device_batch(cfg, "qwen_edit"), "qwen")
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


CASES = dict(kernel_all_codes=kernel_all_codes, kernel_qwen_double=kernel_qwen_double, kernel_flux_single=kernel_flux_single,
             qwen_step_parity=qwen_step_parity, flux_step_parity=flux_step_parity, graph_replay=graph_replay, infer_replay=infer_replay)

if __name__ == "__main__":
    # the step-parity cases run a step under use_deterministic_algorithms(True), where torch allows the modulation-LoRA cuBLAS
    # products only with a fixed workspace configuration (INTEGRATION.md); set before anything initialises cuBLAS here
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    if len(sys.argv) == 2 and sys.argv[1] in CASES:  # one case in this process (tests/test_fp8_weights.py)
        print(CASES[sys.argv[1]]())
    else:
        harness.main(CASES, os.path.abspath(__file__), "fp8_check.log")
