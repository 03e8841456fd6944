"""Activation recompute of the training workspace (DESIGN.md §3): blocks whose saved tensors do not fit keep only their input and
the backward regenerates the rest right before their backward runs.

CPU (emulated kernels, tests/emu_lib.py): the planner, and bit-identical results between keep-all, partially and fully recomputed
plans — in emulation a recompute reproduces the saved tensors exactly, so any difference is a clobbered buffer or a missed entry.
GPU: the recompute reproduces the forward's saved tensors bit for bit at full width, and the reference goldens, graph replay and
the memory the planner promises hold with recompute forced."""
import gc
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import emu_lib
from oracle import mmdit_oracle as mo

HERE = os.path.dirname(os.path.abspath(__file__))
FLUX_YAML = (r"(.*x_embedder|.*transformer_blocks\.[0-9]+\.(norm|norm1)\.linear|.*transformer_blocks\.[0-9]+\.attn\.(to_k|to_q|to_v|to_add_out)"
             r"|.*transformer_blocks\.[0-9]+\.attn\.to_out\.0|.*single_transformer_blocks\.[0-9]+\.attn\.to_out"
             r"|.*single_transformer_blocks\.[0-9]+\.(proj_mlp|proj_out)|.*(?<!single_)transformer_blocks\.[0-9]+\.ff\.net\.2"
             r"|.*(?<!single_)transformer_blocks\.[0-9]+\.ff\.net\.0\.proj|.*(?<!single_)transformer_blocks\.[0-9]+\.norm1_context\.linear"
             r"|.*(?<!single_)transformer_blocks\.[0-9]+\.ff_context\.net\.0\.proj|.*(?<!single_)transformer_blocks\.[0-9]+\.ff_context\.net\.2"
             r"|.*(?<!single_)transformer_blocks\.[0-9]+\.attn\.(to_add_out|add_k_proj|add_q_proj|add_v_proj))")
MODES = ("keep", "partial", "all")


def force_plan(mode):
    """A stand-in for `mmdit_base.plan_activation_memory` that forces a plan: keep-all, the fewest recomputed blocks below keep-all,
    or every block recomputed — chosen through the real planner's own limit."""
    from qflux_b200 import mmdit_base
    real = getattr(mmdit_base.plan_activation_memory, "real", mmdit_base.plan_activation_memory)

    def forced(blocks, fixed, limit):
        p = real(blocks, fixed, None)
        return real(blocks, fixed, {"keep": None, "partial": p.bytes - 1, "all": p.min_bytes}[mode])
    forced.real = real
    return forced


@pytest.fixture()
def emu():
    from qflux_b200 import lib
    restore = emu_lib.install(lib)
    yield lib
    restore()


def _fill(m, seed):
    g = torch.Generator(device=m.dev).manual_seed(seed)
    for k, t in m.w.items():
        if k.endswith("_w") and t.ndim >= 2 and "qknorm" not in k:
            t.normal_(0.0, 0.05, generator=g)
        elif k.endswith("_b"):
            t.normal_(0.0, 0.02, generator=g)
    return m


def _qwen(L=3, targets=("to_q", "to_k", "to_v", "to_out.0"), device="cpu", H=2, J=128):
    from qflux_b200.qwen_model import QwenB200Config, QwenImageB200
    m = QwenImageB200(QwenB200Config(num_layers=L, num_attention_heads=H, joint_attention_dim=J), device=device, _host_only=device == "cpu")
    _fill(m, 7)
    m.add_adapter(4, 8, target_modules=targets, b_std=0.05)
    return m


def _flux(nd=2, ns=3, targets=FLUX_YAML, device="cpu", H=2, J=64, P=64):
    from qflux_b200.flux_model import FluxB200, FluxB200Config
    m = FluxB200(FluxB200Config(num_layers=nd, num_single_layers=ns, attention_head_dim=128, num_attention_heads=H, joint_attention_dim=J,
                                pooled_projection_dim=P, guidance_embeds=True), device=device, _host_only=device == "cpu")
    _fill(m, 11)
    m.add_adapter(4, 4, target_modules=targets, b_std=0.05)
    return m


def _rn(seed):
    g = torch.Generator().manual_seed(seed)
    return lambda *s: torch.randn(*s, generator=g).bfloat16()


def _qwen_batch(kind, seed=0):
    rn = _rn(seed)
    if kind == "dense":
        B, hw, T = 2, 4, 8
        return dict(image_latents=rn(B, 16, 64), control_latents=rn(B, 16, 64), prompt_embeds=rn(B, T, 128) * 3,
                    img_shapes=[[(1, hw, hw), (1, hw, hw)]] * B), rn(B, 16, 64), torch.tensor([0.5, 0.25])
    if kind == "plus":  # Edit-Plus: target + 2 controls of different sizes
        return dict(image_latents=rn(1, 16, 64), control_latents=rn(1, 32, 64), prompt_embeds=rn(1, 16, 128) * 3,
                    img_shapes=[[(1, 4, 4), (1, 4, 6), (1, 2, 4)]]), rn(1, 16, 64), torch.tensor([0.25])
    # pad-to-max multi-resolution batch whose padding spans whole 256-row bands (ragged GEMM row bands) and padded text
    shapes = [[(1, 24, 16), (1, 24, 16)], [(1, 8, 8), (1, 8, 8)], [(1, 16, 16), (1, 16, 16)]]
    lt = [sh[0][1] * sh[0][2] for sh in shapes]
    B, T, txt, Lt = 3, 8, [8, 5, 7], max(lt)
    x0, ctrl, pe, noise = rn(B, Lt, 64), rn(B, Lt, 64), rn(B, T, 128) * 3, rn(B, Lt, 64)
    mask = torch.zeros(B, T, dtype=torch.int64)
    for b in range(B):
        x0[b, lt[b]:] = 0
        ctrl[b, lt[b]:] = 0
        noise[b, lt[b]:] = 0
        pe[b, txt[b]:] = 0
        mask[b, :txt[b]] = 1
    return dict(image_latents=x0, control_latents=ctrl, prompt_embeds=pe, prompt_embeds_mask=mask, img_shapes=shapes), noise, torch.tensor([0.5, 0.25, 0.75])


def _flux_batch(kind, seed=0):
    from qflux_b200.train_step import FluxKontextStep
    rn = _rn(seed)
    T = 8
    if kind == "dense":
        B, hw = 2, 4
        return dict(image_latents=rn(B, 16, 64), control_latents=rn(B, 16, 64), pooled_prompt_embeds=rn(B, 64), prompt_embeds=rn(B, T, 64),
                    text_ids=torch.zeros(T, 3), image_ids=FluxKontextStep.latent_image_ids(hw, hw, "cpu", 0.0),
                    control_ids=FluxKontextStep.latent_image_ids(hw, hw, "cpu", 1.0)), rn(B, 16, 64), torch.tensor([0.5, 0.25])
    shapes = [[(1, 16, 16), (1, 16, 16)], [(1, 8, 4), (1, 4, 8)], [(1, 8, 8), (1, 4, 4), (1, 4, 8)]]
    lt = [sh[0][1] * sh[0][2] for sh in shapes]
    lc = [sum(h * w for (_, h, w) in sh[1:]) for sh in shapes]
    B, Lm, Lcm = 3, max(lt), max(lc)
    x0, ctrl, noise = rn(B, Lm, 64), rn(B, Lcm, 64), rn(B, Lm, 64)
    for b in range(B):
        x0[b, lt[b]:] = 0
        noise[b, lt[b]:] = 0
        ctrl[b, lc[b]:] = 0
    return dict(image_latents=x0, control_latents=ctrl, pooled_prompt_embeds=rn(B, 64), prompt_embeds=rn(B, T, 64), text_ids=torch.zeros(T, 3),
                img_shapes=shapes), noise, torch.tensor([0.5, 0.25, 0.125])


def _step(m, family, loss_kind="mse", **kw):
    from qflux_b200.train_step import FluxKontextStep, QwenImageEditStep
    return (QwenImageEditStep if family == "qwen" else FluxKontextStep)(m, loss_kind, **kw)


def _fused(m, family, batch, loss_kind="mse"):
    """loss, prediction and the flat fp32 LoRA gradient of one fused step (train_step's recipe without the optimizer)."""
    emb, noise, u = batch
    step = _step(m, family, loss_kind)
    loss = step._run(*step._prepare(emb, noise, u))
    return float(loss), m._ws["pred"].clone(), m.G32.clone()


def _same(a, b):
    assert a[0] == b[0]
    for x, y in zip(a[1:], b[1:]):
        assert torch.equal(x, y)


def _across_plans(monkeypatch, make, run, expect_partial=True):
    """run(make()) under the three plans; returns the keep-all result after checking the other two against it bit for bit."""
    from qflux_b200 import mmdit_base
    res, plans = {}, {}
    for mode in MODES:
        monkeypatch.setattr(mmdit_base, "plan_activation_memory", force_plan(mode))
        m = make()
        res[mode] = run(m)
        plans[mode] = m.activation_plan
    assert plans["keep"].recompute == () and plans["keep"].saved_bytes == 0
    assert plans["all"].recompute == tuple(range(m.L + m.Ls))
    if expect_partial:
        assert 0 < len(plans["partial"].recompute) < len(plans["all"].recompute)
    for mode in ("partial", "all"):
        _same(res["keep"], res[mode])
    return res["keep"]


# ------------------------------------------------------------------------------------------------------------------ planner
def test_planner_keeps_everything_when_it_fits():
    from qflux_b200.mmdit_base import plan_activation_memory
    blocks = [("dbl", {"a": 10, "b": 5})] * 4
    p = plan_activation_memory(blocks, 100, 160)
    assert p.recompute == () and p.bytes == 160 and p.saved_bytes == 0 and p.min_bytes == 115
    assert plan_activation_memory(blocks, 100, None).recompute == ()


def test_planner_recomputes_the_fewest_blocks_from_the_end():
    from qflux_b200.mmdit_base import plan_activation_memory
    blocks = [("dbl", {"a": 10})] * 6
    # one recomputed block needs a scratch as large as itself: the first saving comes with the second block
    p = plan_activation_memory(blocks, 0, 59)
    assert p.recompute == (4, 5) and p.bytes == 50 and p.saved_bytes == 10
    assert plan_activation_memory(blocks, 0, 30).recompute == (2, 3, 4, 5)
    assert plan_activation_memory(blocks, 0, 10).recompute == tuple(range(6))


def test_planner_mixed_double_and_single_blocks():
    from qflux_b200.mmdit_base import plan_activation_memory
    # two double blocks (one with an optional entry), then three single blocks of a smaller size
    blocks = [("dbl", {"a": 20, "h": 8}), ("dbl", {"a": 20})] + [("sgl", {"c": 12, "y": 3})] * 2 + [("sgl", {"c": 12})]
    keep = 28 + 20 + 15 + 15 + 12
    assert plan_activation_memory(blocks, 0, None).bytes == keep
    p = plan_activation_memory(blocks, 0, keep - 1)  # singles first; the scratch holds every entry its blocks need (c and y)
    assert p.recompute == (3, 4) and p.bytes == keep - 15 - 12 + 15
    p = plan_activation_memory(blocks, 0, 70)
    assert p.recompute == (2, 3, 4) and p.bytes == 28 + 20 + 15
    p = plan_activation_memory(blocks, 0, 62)  # four blocks would take 28 + 20 (double scratch) + 15: only all five fit
    assert p.recompute == (0, 1, 2, 3, 4) and p.bytes == p.min_bytes == 28 + 15
    p = plan_activation_memory(blocks, 0, 28 + 15)
    assert p.recompute == (0, 1, 2, 3, 4) and p.bytes == p.min_bytes == 28 + 15


def test_planner_raises_when_nothing_fits():
    from qflux_b200 import lib
    from qflux_b200.mmdit_base import plan_activation_memory
    with pytest.raises(lib.QfxError, match=r"needs 1015 bytes with the activations of every block recomputed, but only 1014 bytes"):
        plan_activation_memory([("dbl", {"a": 10, "b": 5})] * 4, 1000, 1014)


def test_host_only_models_are_unlimited(emu):
    m = _qwen()
    assert m._activation_limit_now() is None
    emb, noise, u = _qwen_batch("dense")
    _fused(m, "qwen", (emb, noise, u))
    assert m.activation_plan.recompute == () and m.activation_plan.limit is None


def _ws_bytes(ws):
    seen, total = set(), 0

    def walk(v):
        nonlocal total
        if torch.is_tensor(v):
            st = v.untyped_storage()
            if st.data_ptr() not in seen:
                seen.add(st.data_ptr())
                total += st.nbytes()
        elif isinstance(v, dict):
            for x in v.values():
                walk(x)
        elif isinstance(v, (list, tuple)):
            for x in v:
                walk(x)
    walk(ws)
    return total


@pytest.mark.parametrize("family", ["qwen", "flux"])
@pytest.mark.parametrize("mode", MODES)
def test_planned_bytes_are_the_allocated_bytes(emu, monkeypatch, family, mode):
    from qflux_b200 import mmdit_base
    monkeypatch.setattr(mmdit_base, "plan_activation_memory", force_plan(mode))
    m = _qwen(4, ("to_q", "img_mlp.net.2", "img_mod.1", "txt_in")) if family == "qwen" else _flux()
    ws = m._workspace(2, 8, 32, True)
    assert _ws_bytes(ws) == ws["plan"].bytes
    if mode != "keep":  # every recomputed block of a kind shares one dict
        rec = ws["plan"].recompute
        dicts = [ws["dbl"][b] if b < m.L else ws["sgl"][b - m.L] for b in rec]
        assert len({id(d) for d in dicts}) == len({b < m.L for b in rec})


def test_changing_the_limit_rebuilds_the_workspace(emu):
    m = _qwen(4)
    batch = _qwen_batch("dense")
    r0 = _fused(m, "qwen", batch)
    p0, ws0 = m.activation_plan, m._ws
    assert p0.recompute == ()
    m.set_activation_memory_limit(p0.min_bytes)
    assert m.activation_plan is None
    r1 = _fused(m, "qwen", batch)
    assert m._ws is not ws0 and m.activation_plan.recompute == (0, 1, 2, 3) and m.activation_plan.limit == p0.min_bytes
    m.set_activation_memory_limit(p0.bytes - 1)
    r2 = _fused(m, "qwen", batch)
    assert m.activation_plan.recompute == (2, 3)
    m.set_activation_memory_limit(None)
    r3 = _fused(m, "qwen", batch)
    assert m.activation_plan.recompute == ()
    for r in (r1, r2, r3):
        _same(r0, r)
    from qflux_b200 import lib
    m.set_activation_memory_limit(p0.min_bytes - 1)
    with pytest.raises(lib.QfxError, match="every block recomputed"):
        _fused(m, "qwen", batch)


# ------------------------------------------------------------------------------------------------------------------ bit-identical plans
@pytest.mark.parametrize("case", ["qwen_dense", "qwen_plus3", "qwen_multires", "flux_dense", "flux_multires"])
def test_plans_give_identical_steps(emu, monkeypatch, case):
    family, kind = case.split("_")
    if family == "qwen":
        make = lambda: _qwen(4, ("to_q", "to_k", "to_v", "to_out.0", "img_mlp.net.2"))
        batch = _qwen_batch("multires" if kind == "multires" else kind)
    else:
        make = lambda: _flux(2, 3, FLUX_YAML if kind == "dense" else ("to_q", "to_k", "to_v", "to_out.0", "proj_mlp", "ff.net.2"))
        batch = _flux_batch(kind)
    loss_kind = "attention_mask" if kind == "multires" else "mse"
    out = _across_plans(monkeypatch, make, lambda m: _fused(m, family, batch, loss_kind))
    assert out[2].abs().sum() > 0


@pytest.mark.parametrize("targets", [("to_q", "img_mlp.net.2", "txt_mlp.net.2"),   # ff.net.2: the kept MLP activation `h`
                                     ("to_k", "img_mod.1", "txt_mod.1"),            # AdaLN linears: the un-gated outputs y_attn / y_mlp
                                     ("to_v", "img_in", "txt_in")])                 # the embedders (outside the blocks)
def test_qwen_lora_sites_across_plans(emu, monkeypatch, targets):
    batch = _qwen_batch("dense", seed=3)
    out = _across_plans(monkeypatch, lambda: _qwen(4, targets), lambda m: _fused(m, "qwen", batch))
    assert out[2].abs().sum() > 0


@pytest.mark.parametrize("targets", [r".*(ff\.net\.2|attn\.to_q)",
                                     r".*(norm1\.linear|norm1_context\.linear|single_transformer_blocks\.[0-9]+\.norm\.linear|attn\.to_k)",
                                     r".*(x_embedder|context_embedder|single_transformer_blocks\.[0-9]+\.(proj_out|proj_mlp))"])
def test_flux_lora_sites_across_plans(emu, monkeypatch, targets):
    batch = _flux_batch("dense", seed=4)
    out = _across_plans(monkeypatch, lambda: _flux(2, 3, targets), lambda m: _fused(m, "flux", batch))
    assert out[2].abs().sum() > 0


@pytest.mark.parametrize("family", ["qwen", "flux"])
def test_gradient_accumulation_across_plans(emu, monkeypatch, family):
    batches = [(_qwen_batch if family == "qwen" else _flux_batch)("dense", seed=s) for s in (5, 6)]

    def run(m):
        step = _step(m, family, gradient_accumulation_steps=2, use_cuda_graph=False)
        losses = [float(step.train_step(emb, None, noise, u)) for emb, noise, u in batches]
        return losses[0] + 1000 * losses[1], m.G32.clone(), m.G16.clone()
    _across_plans(monkeypatch, lambda: _qwen(4) if family == "qwen" else _flux(), run)


@pytest.mark.parametrize("family", ["qwen", "flux"])
def test_autograd_bridges_across_plans(emu, monkeypatch, family):
    batch = (_qwen_batch if family == "qwen" else _flux_batch)("dense", seed=8)
    emb, noise, u = batch

    def run(m):
        step = _step(m, family)
        loss = step.compute_loss(emb, noise=noise, u=u) if family == "qwen" else step.compute_loss(emb, noise=noise, t=u)
        loss.backward()
        grads = torch.cat([p.grad.float().reshape(-1) for p in m.parameters()])
        return loss.item(), m._ws["pred"].clone(), grads
    _across_plans(monkeypatch, lambda: _qwen(4, ("to_q", "img_mod.1", "txt_in")) if family == "qwen" else _flux(), run)

    if family == "qwen":  # the module forward's autograd bridge (ModelFn)
        def run_module(m):
            hs = torch.cat([emb["image_latents"], emb["control_latents"]], 1)
            out = m(hidden_states=hs, encoder_hidden_states=emb["prompt_embeds"], timestep=torch.tensor([0.5, 0.25]),
                    img_shapes=emb["img_shapes"])[0]
            (out.float() ** 2).sum().backward()
            return 0.0, out.detach().clone(), torch.cat([p.grad.float().reshape(-1) for p in m.parameters()])
        _across_plans(monkeypatch, lambda: _qwen(4, ("to_q", "img_mod.1", "txt_in")), run_module)


# ------------------------------------------------------------------------------------------------------------------ sharded (gloo)
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker_sharded(rank, world, port, out):
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.dirname(HERE))
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "qwen-image-finetune_b200"))
    import emu_lib as el
    from qflux_b200 import lib
    el.install(lib)
    import test_activation_recompute as t
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    ok = {}
    for family in ("qwen", "flux"):
        make = (lambda: t._qwen(3, ("to_q", "to_out.0", "img_mod.1", "net.2"))) if family == "qwen" else (lambda: t._flux(3, 3, FLUX_YAML))
        batch = (t._qwen_batch if family == "qwen" else t._flux_batch)("dense", seed=100 + rank)
        full = t._fused(make(), family, batch)
        sh = make().shard_frozen_weights()
        probe = t._fused(sh, family, batch)
        sh.set_activation_memory_limit(sh.activation_plan.min_bytes)
        rec = [t._fused(sh, family, batch) for _ in range(2)]  # the second step starts from the rings as the first backward left them
        ok[family] = dict(keep=probe[0] == full[0] and torch.equal(probe[2], full[2]),
                          n_rec=len(sh.activation_plan.recompute), n=sh.L + sh.Ls,
                          same=all(r[0] == full[0] and torch.equal(r[1], full[1]) and torch.equal(r[2], full[2]) for r in rec))
    allr = [None] * world
    dist.all_gather_object(allr, ok)
    if rank == 0:
        torch.save(allr, out)
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_sharded_recompute_matches_replicated_keep_all(tmp_path):
    out = str(tmp_path / "res.pt")
    mp.spawn(_worker_sharded, args=(2, _free_port(), out), nprocs=2, join=True)
    for r in torch.load(out):
        for fam, v in r.items():
            assert v["keep"] and v["same"] and v["n_rec"] == v["n"], (fam, v)


# ------------------------------------------------------------------------------------------------------------------ GPU
def _gpu_model(family):
    """6 full-width blocks (D = 3072, 24 heads) with the benchmark adapters."""
    if family == "qwen":
        return _qwen(6, ("to_q", "to_k", "to_v", "to_out.0", "img_mod.1", "img_mlp.net.2"), device="cuda", H=24, J=3584)
    return _flux(3, 3, FLUX_YAML, device="cuda", H=24, J=4096, P=768)


def _gpu_batch(family, B=1, seed=0):
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g).bfloat16().cuda()
    if family == "qwen":
        return dict(image_latents=rn(B, 1024, 64), control_latents=rn(B, 1024, 64), prompt_embeds=rn(B, 352, 3584) * 3,
                    img_shapes=[[(1, 32, 32), (1, 32, 32)]] * B), rn(B, 1024, 64), torch.rand(B, generator=g)
    from qflux_b200.train_step import FluxKontextStep
    return dict(image_latents=rn(B, 1024, 64), control_latents=rn(B, 1024, 64), pooled_prompt_embeds=rn(B, 768), prompt_embeds=rn(B, 512, 4096),
                text_ids=torch.zeros(512, 3), image_ids=FluxKontextStep.latent_image_ids(32, 32, "cpu", 0.0),
                control_ids=FluxKontextStep.latent_image_ids(32, 32, "cpu", 1.0)), rn(B, 1024, 64), torch.rand(B, generator=g).bfloat16()


def _same_loss(a, b):
    """The loss is an fp32 sum that the flow-loss kernel reduces across CTAs with atomics: its last bits depend on their order."""
    assert abs(a - b) <= 1e-6 * abs(b), (a, b)


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["qwen", "flux"])
def test_recompute_reproduces_the_saved_tensors(family):
    """The scratch at entry to a recomputed block's backward equals that block's own saved dict of a keep-all run, entry for entry."""
    m = _gpu_model(family)
    batch = _gpu_batch(family)
    blk = 1  # a double block; for FLUX also the first single block
    snaps = {}

    def hook(name, orig, which):
        def f(ws, l, *a):
            if l == which:
                save = a[-3] if name == "dbl" else a[-2]
                snaps.setdefault(mode, {})[name] = {k: v.clone() for k, v in save.items()}
                snaps[mode][name + "_loraT"] = {k: v.clone() for k, v in ws["loraT"].items() if k[0] == l and k[1].startswith("s_") == (name == "sgl")}
            return orig(ws, l, *a)
        return f
    res = {}
    m._double_bwd = hook("dbl", type(m)._double_bwd.__get__(m), blk)
    if m.Ls:
        m._single_bwd = hook("sgl", type(m)._single_bwd.__get__(m), 0)
    for mode in ("keep", "all"):
        m.set_activation_memory_limit(1 << 62 if mode == "keep" else res["keep"][3].min_bytes)
        loss, pred, g = _fused(m, family, batch)
        res[mode] = (loss, pred, g, m.activation_plan)
    assert res["keep"][3].recompute == () and len(res["all"][3].recompute) == m.L + m.Ls
    for name in snaps["keep"]:
        a, b = snaps["keep"][name], snaps["all"][name]
        assert set(a) == set(b), name
        for k in a:
            assert torch.equal(a[k], b[k]), (name, k)
    _same_loss(res["all"][0], res["keep"][0])
    assert torch.equal(res["keep"][1], res["all"][1])
    d = _rel(res["all"][2], res["keep"][2])
    print(f"{family}: LoRA gradient, recompute vs keep-all: rel L2 {d:.2e}")
    assert d < 1e-2


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["qwen_hd128", "qwen_hd128_plus3", "qwen_hd128_alltargets", "qwen_hd128_editmask", "flux_hd128",
                                  "flux_hd128_yaml", "flux_custom_multires", "qwen_custom_multires"])
def test_reference_goldens_with_recompute(monkeypatch, name):
    import test_reference_goldens as trg
    from qflux_b200 import mmdit_base
    monkeypatch.setattr(mmdit_base, "plan_activation_memory", force_plan("all"))
    trg._b200_step(name, "cuda", False, 2e-2, 3e-2)


@pytest.mark.gpu
@pytest.mark.parametrize("family", ["qwen", "flux"])
def test_graph_replay_with_recompute_equals_eager(family):
    m = _gpu_model(family)
    emb, noise, u = _gpu_batch(family, seed=2)
    _fused(m, family, (emb, noise, u))
    m.set_activation_memory_limit(m.activation_plan.min_bytes)
    step = _step(m, family)
    outs = []
    for _ in range(3):  # eager, capture + first replay, replay
        outs.append((float(step._graphs.run(m, step._run, step._prepare(emb, noise, u), tag=False)), m._ws["pred"].clone()))
    assert step._graphs.captured() == 1 and len(m.activation_plan.recompute) == m.L + m.Ls
    for loss, pred in outs[1:]:
        _same_loss(loss, outs[0][0])
        assert torch.equal(pred, outs[0][1])


@pytest.mark.gpu
def test_recompute_lowers_peak_memory_by_what_the_plan_saves():
    m = _gpu_model("qwen")
    batch = _gpu_batch("qwen", B=4, seed=3)
    peaks = {}
    for mode in ("keep", "all"):
        if mode == "all":
            m.set_activation_memory_limit(plan.min_bytes)
        gc.collect()  # models of earlier tests must not be freed inside one of the two measurements
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        _fused(m, "qwen", batch)
        torch.cuda.synchronize()
        peaks[mode] = torch.cuda.max_memory_allocated() - base
        plan = m.activation_plan
    saved = plan.saved_bytes
    print(f"planned saving {saved / 2**30:.2f} GiB, measured {(peaks['keep'] - peaks['all']) / 2**30:.2f} GiB")
    assert saved > 0 and peaks["keep"] - peaks["all"] >= 0.9 * saved
