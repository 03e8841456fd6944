"""LoRA ranks other than 4/8/16/32/64: any multiple of 4 from 4 to 128, one rank for every adapted module.  Above 64 the factors are
padded to two 64-wide k-blocks (Rp = 128).

CPU:
  * the oracle reproduces the reference's own vectors at r = 24, 96 and 128 (tests/golden/ref_rank_golden_*.pt, rank_cases.py);
  * the fused host path with emulated kernels (tests/emu_wide.py over tests/emu_lib.py) reproduces them at DESIGN.md §2's tolerances, every LoRA gradient tensor on its own;
  * tests/emu_wide.py's weight gradient agrees with fp64 at r up to 128 and with tests/emu_lib.py's at r <= 64;
  * add_adapter refuses a rank outside the rule, and per-module patterns, before anything is allocated;
  * load_lora_adapter round-trips a saved r = 96 file;
  * at r = 16 the step calls the same entry points with the same shapes, k-blocks and ranks as before wider ranks existed
    (tests/golden/lib_calls_r16.json, recorded from the host code that took r in 4/8/16/32/64 only).
GPU (`-m gpu`): the CUDA path against the same goldens; tools/wide_rank_check.py per element against fp64 (the weight-gradient kernels
at r up to 128, the fused GEMM at kb2 = 2), two deterministic r = 128 steps bit for bit, CUDA-graph replay at r = 128 under both
settings of the deterministic flag, and a 5-step AdamW trajectory at r = 128 against the fp32 oracle."""
import json
import os
import subprocess
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, HERE)
import rank_cases  # noqa: E402
import ref_common as rc  # noqa: E402

CALLS = os.path.join(HERE, "golden", "lib_calls_r16.json")
CHECK = os.path.join(ROOT, "tools", "wide_rank_check.py")
_G = {}


def golden():
    if not _G:
        _G.update(rank_cases.load(os.path.join(HERE, "golden"), "ref_rank_golden"))
    return _G


def _b200_model(spec, device, host_only):
    from test_reference_goldens import _b200_model as build
    return build(spec, device, host_only)


def fused_step(spec, c, device, host_only):
    """(model, pred [B, L, 64] fp32 on the host, loss) of one fused training step on a stored case's inputs (Qwen / FLUX, shared mode)."""
    from qflux_b200.train_step import FluxKontextStep, QwenImageEditStep
    m, chk = _b200_model(spec, device, host_only)
    x, ex = c["inputs"], c["extra"]
    bf = lambda t: t.to(device).bfloat16()
    if spec["kind"] == "qwen":
        step = QwenImageEditStep(m, use_cuda_graph=False)
        emb = dict(image_latents=bf(x["image_latents"]), control_latents=bf(x["control_latents"]), prompt_embeds=bf(x["prompt_embeds"]),
                   img_shapes=[[tuple(s) for s in sh] for sh in x["img_shapes"]])
        loss = step.compute_loss(emb, noise=bf(ex["noise"]), u=ex["u"])
    else:
        step = FluxKontextStep(m, use_cuda_graph=False)
        emb = dict(image_latents=bf(x["image_latents"]), control_latents=bf(x["control_latents"]),
                   pooled_prompt_embeds=bf(x["pooled_prompt_embeds"]), prompt_embeds=bf(x["prompt_embeds"]), text_ids=x["text_ids"],
                   image_ids=ex["image_ids"], control_ids=ex["control_ids"])
        loss = step.compute_loss(emb, noise=bf(x["noise"]), t=x["timestep"])
    pred = m._ws["pred"].view(c["pred"].shape[0], -1, 64).float().cpu().clone()
    loss.backward()
    return m, chk, pred, loss


def check_against_golden(name, device, host_only):
    spec, c = rank_cases.RANK_CASES[name], golden()[name]
    m, chk, pred, loss = fused_step(spec, c, device, host_only)
    assert abs(chk - c["weight_checksum"]) <= 1e-9 * c["weight_checksum"], "fused state-dict key set differs from the reference's"
    assert m.lora_rank == spec["r"] and m.lora_rp == 64 * -(-spec["r"] // 64)
    Lq = c["inputs"]["image_latents"].shape[1]
    assert rc.rel_l2(pred[:, :Lq], c["pred"][:, :Lq]) < 2e-2, rc.rel_l2(pred[:, :Lq], c["pred"][:, :Lq])
    assert abs(loss.item() - c["loss"].item()) < 1e-2 * max(1.0, abs(c["loss"].item()))
    grads = {n: p.grad.float().cpu() for n, p in m.named_parameters()}
    assert sorted(grads) == sorted(c["grads"])
    worst = max((rc.rel_l2(grads[n], ref), n) for n, ref in c["grads"].items() if ref.norm() > 0)
    assert worst[0] < 3e-2, worst
    for n, ref in c["grads"].items():
        if ref.norm() == 0:
            assert grads[n].norm() == 0, n


# ------------------------------------------------------------------------------------------------------------------ goldens
@pytest.mark.parametrize("name", list(rank_cases.RANK_CASES))
def test_oracle_matches_reference_at_wide_ranks(name):
    from oracle import mmdit_oracle as mo
    from test_reference_goldens import _oracle
    spec, c = rank_cases.RANK_CASES[name], golden()[name]
    orc, chk = _oracle(spec)
    assert sum(p.numel() for p in orc.parameters()) == c["n_params"]
    assert abs(chk - c["weight_checksum"]) <= 1e-9 * c["weight_checksum"]
    assert sorted(n for n, p in orc.named_parameters() if p.requires_grad) == c["lora_keys"]
    x, ex = c["inputs"], c["extra"]
    if spec["kind"] == "qwen":
        shapes = [[tuple(s) for s in sh] for sh in x["img_shapes"]]
        loss, pred = mo.qwen_compute_loss(orc, x["image_latents"], x["control_latents"], x["prompt_embeds"], x["prompt_embeds_mask"], shapes,
                                          noise=ex["noise"], u=ex["u"])
    else:
        loss, pred = mo.flux_compute_loss_shared(orc, x["image_latents"], x["control_latents"], x["pooled_prompt_embeds"], x["prompt_embeds"],
                                                 x["text_ids"], ex["image_ids"], ex["control_ids"], noise=x["noise"], t=x["timestep"])
    loss.backward()
    ref_pred = c["pred"][:, : pred.shape[1]]
    assert rc.rel_l2(pred.detach(), ref_pred) < 1e-5, rc.rel_l2(pred.detach(), ref_pred)
    assert abs(loss.item() - c["loss"].item()) < 1e-5
    for n, p in orc.named_parameters():
        if p.requires_grad:
            g = p.grad if p.grad is not None else torch.zeros_like(p)
            ref = c["grads"][n]
            assert (g - ref).norm() <= 1e-5 * ref.norm() + 1e-7, (n, rc.rel_l2(g, ref))


@pytest.mark.parametrize("name", list(rank_cases.RANK_CASES))
def test_emulated_path_matches_reference_at_wide_ranks(name):
    import emu_wide
    from qflux_b200 import lib
    restore = emu_wide.install(lib)
    try:
        check_against_golden(name, "cpu", True)
    finally:
        restore()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(rank_cases.RANK_CASES))
def test_cuda_path_matches_reference_at_wide_ranks(name):
    check_against_golden(name, "cuda", False)


def test_wide_emulation_agrees_with_fp64_and_with_emu_lib():
    import emu_lib
    import emu_wide
    import wide_rank_check as wc
    torch.manual_seed(0)
    M, Dg = 77, 128
    for r in (1, 24, 64, 68, 96, 128):
        rp = 64 * -(-r // 64)
        for G in (1, 2, 3):
            B = torch.randn(M, rp * G).bfloat16()
            for mode, Na in ((0, 256), (1, G * Dg)):
                A = torch.randn(M, Na).bfloat16()
                rows = Dg if mode else Na
                Gs = [torch.zeros(rows * r) for _ in range(G)]
                emu_wide.lora_wgrad_tc(A, B, Gs, 1, rows, r, mode=mode, Dg=Dg)
                for g, (ref, mag) in enumerate(wc.wgrad_ref(A, B, r, G, mode, Dg)):
                    got = torch.as_strided(Gs[g], (rows, r), (1, rows)).double()
                    assert ((got - ref).abs() <= 1e-5 * mag + 1e-30).all(), (r, G, mode, g)
                if r <= 64:
                    Ge = [torch.zeros(rows * r) for _ in range(G)]
                    emu_lib.lora_wgrad_tc(A, B, Ge, 1, rows, r, mode=mode, Dg=Dg)
                    assert all(torch.equal(a, b) for a, b in zip(Gs, Ge))


# ------------------------------------------------------------------------------------------------------------------ rank rule
def _host_qwen():
    from qflux_b200.qwen_model import QwenB200Config, QwenImageB200
    return QwenImageB200(QwenB200Config(num_layers=1, num_attention_heads=1, joint_attention_dim=128), device="cpu", _host_only=True)


@pytest.mark.parametrize("r", [2, 126, 132, 0, -4, 256])
def test_add_adapter_refuses_ranks_outside_the_rule(r, monkeypatch):
    from qflux_b200 import mmdit_base
    m = _host_qwen()

    def no_alloc(*a, **k):
        raise AssertionError("allocated before the rank was checked")
    monkeypatch.setattr(mmdit_base.LoraSite, "__init__", no_alloc)
    monkeypatch.setattr(mmdit_base.torch, "zeros", no_alloc)
    with pytest.raises(NotImplementedError, match="multiple of 4 from 4 to 128"):
        m.add_adapter(r, r)
    cfg = mmdit_base._LoraConfigLike(r=r, lora_alpha=16, target_modules=["to_q"])
    with pytest.raises(NotImplementedError, match="multiple of 4 from 4 to 128"):
        m.add_adapter(cfg)
    assert not m._lora_params and not m.sites and m.G32 is None and m.lora_rank == 0


def test_add_adapter_refuses_per_module_patterns_before_allocating(monkeypatch):
    from qflux_b200 import mmdit_base
    m = _host_qwen()
    monkeypatch.setattr(mmdit_base.torch, "zeros", lambda *a, **k: (_ for _ in ()).throw(AssertionError("allocated")))
    for attr in ("rank_pattern", "alpha_pattern"):
        cfg = mmdit_base._LoraConfigLike(r=96, lora_alpha=96, target_modules=["to_q"])
        setattr(cfg, attr, {"to_q": 8})
        with pytest.raises(NotImplementedError, match="per-module rank / alpha"):
            m.add_adapter(cfg)
    assert not m._lora_params and not m.sites and m.G32 is None


@pytest.mark.parametrize("r", [4, 12, 24, 60, 64, 68, 96, 124, 128])
def test_every_rank_of_the_rule_lays_out_its_factors(r):
    from qflux_b200.mmdit_base import rank_chunks
    m = _host_qwen().add_adapter(r, 2 * r, target_modules=["to_q", "to_k", "to_out.0", "img_in"], b_std=0.05)
    rp = 64 * -(-r // 64)
    assert m.lora_rp == rp
    for site in m._unique_sites():
        assert site.rp == rp and site.A_pad.shape[0] == site.n * rp and site.B_pad.shape[1] == rp
        for slot, (full, pA, pB, *_rest) in site.members.items():
            assert pA.shape[0] == r and pB.shape[1] == r and pB.stride(0) == rp
            assert pA.data_ptr() == site.A_pad[slot * rp].data_ptr()
        assert not site.A_pad.view(site.n, rp, -1)[:, r:].any() and not site.B_pad[:, r:].any()
    chunks = rank_chunks(r)
    assert sum(w for _, w in chunks) == r and all(w in (4, 8, 16, 32, 64) for _, w in chunks)
    assert all(c0 % 8 == 0 for c0, _ in chunks) and [c0 for c0, _ in chunks] == sorted(c0 for c0, _ in chunks)
    assert [w for _, w in chunks] == sorted((w for _, w in chunks), reverse=True)


def test_load_lora_adapter_round_trips_an_r96_file(tmp_path):
    import safetensors.torch
    targets = ["to_q", "to_k", "to_v", "to_out.0", "img_mod.1", "img_in"]
    src = _host_qwen().add_adapter(96, 96, target_modules=targets, b_std=0.05, seed=3)
    lora = {f"transformer.{k.replace('.default.', '.')}": v for k, v in src.state_dict().items() if ".lora_" in k}
    path = tmp_path / "pytorch_lora_weights.safetensors"
    safetensors.torch.save_file(lora, str(path))
    dst = _host_qwen()
    dst.load_lora_adapter(str(tmp_path))
    assert dst.lora_rank == 96 and dst.lora_rp == 128 and dst.lora_scaling == 1.0
    a, b = src.state_dict(), dst.state_dict()
    keys = [k for k in a if ".lora_" in k]
    assert sorted(keys) == sorted(k for k in b if ".lora_" in k)
    for k in keys:
        assert torch.equal(a[k], b[k]), k
    for site in dst._unique_sites():  # the padding past r stays zero
        assert not site.A_pad.view(site.n, 128, -1)[:, 96:].any() and not site.B_pad[:, 96:].any()


# ------------------------------------------------------------------------------------------------------------------ r = 16 unchanged
def _desc(t):
    return None if t is None else [list(t.shape), list(t.stride()), t.storage_offset()]


def record_calls():
    """Every gemm / weight-gradient call of one emulated training step (flag off and on) of a Qwen model with LoRA on every Linear
    the fused path adapts (img_in: the narrow embedder path) and a FLUX model with BASELINE config 3's targets, at r = 16: the
    entry point, its shape arguments, each operand's shape / strides / offset, kb2, a2_col0 and r; plus the LoRA buffer shapes."""
    import det_ref
    import emu_wide
    from qflux_b200 import lib
    log = []
    restore = emu_wide.install(lib, det_ref.install)
    saved = {n: getattr(lib, n) for n in ("gemm", "lora_wgrad_tc", "lora_wgrad", "lora_wgrad_tc_det", "lora_wgrad_det")}

    def gemm(probs, N, K, **kw):
        log.append(["gemm", N, K, sorted(kw.items()), [[_desc(p.A), _desc(p.B), _desc(p.out), _desc(p.A2), _desc(p.B2), p.kb2, p.a2_col0]
                                                       for p in probs]])
        return saved["gemm"](probs, N, K, **kw)

    def wgrad(name):
        def f(A, B, G, gs_i, gs_j, r, *a, **kw):
            Gs = G if isinstance(G, list) else [G]
            log.append([name, _desc(A), _desc(B), [g.storage_offset() for g in Gs], gs_i, gs_j, r, list(a),
                        sorted((k, v) for k, v in kw.items() if k != "scratch"), kw["scratch"].numel() if "scratch" in kw else None])
            return saved[name](A, B, G, gs_i, gs_j, r, *a, **kw)
        return f
    lib.gemm = gemm
    for n in ("lora_wgrad_tc", "lora_wgrad", "lora_wgrad_tc_det", "lora_wgrad_det"):
        setattr(lib, n, wgrad(n))
    was = torch.are_deterministic_algorithms_enabled()
    try:
        cases = [("qwen", dict(rank_cases.RANK_CASES["qwen_hd128_r24"], r=16, targets=rc.QWEN_ALL_TARGETS), "qwen_hd128_r24"),
                 ("flux", dict(rank_cases.RANK_CASES["flux_hd128_yaml_r96"], r=16), "flux_hd128_yaml_r96")]
        for tag, spec, gname in cases:
            for det in (False, True):
                torch.use_deterministic_algorithms(det)
                log.append(["case", tag, det])
                m, *_ = fused_step(spec, golden()[gname], "cpu", True)
                log.append(["buffers", [[list(s.A_pad.shape), list(s.B_pad.shape)] for s in m._unique_sites()],
                            sorted([list(k), list(v.shape)] for k, v in m._ws["loraT"].items()), list(m._ws["U"].shape),
                            list(m._gscratch.shape), list(m.G32.shape), list(m._ws["det_scratch"].shape) if det else None])
    finally:
        torch.use_deterministic_algorithms(was)
        for n, f in saved.items():
            setattr(lib, n, f)
        restore()
    return json.loads(json.dumps(log))


def test_r16_calls_are_unchanged():
    with open(CALLS) as f:
        want = json.load(f)
    got = record_calls()
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g == w, (i, g, w)


# ------------------------------------------------------------------------------------------------------------------ GPU
def _run_check(name):
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8")
    r = subprocess.run([sys.executable, CHECK, "--case", name], capture_output=True, text=True, timeout=1200, env=env, cwd=ROOT)
    res = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
    assert r.returncode == 0 and res, (r.stdout + r.stderr)[-3000:]
    out = json.loads(res[-1][7:])
    print(f"WIDE_RANK {name} " + json.dumps(out))
    return out


def _gpu_cases():
    import wide_rank_check
    return list(wide_rank_check.CASES)


@pytest.mark.gpu
@pytest.mark.parametrize("name", _gpu_cases())
def test_wide_rank_gpu_case(name):
    r = _run_check(name)
    assert not r["fail"], r["fail"][:20]
