"""Bit-reproducible data-parallel steps on one host: under torch.use_deterministic_algorithms(True) the flat LoRA gradient of the ranks
is summed in rank order through peer memory (qflux_b200/sharding.py GradExchange, qfx_dp_reduce_det) instead of an NCCL all-reduce.

CPU (emulated kernels, tests/emu_lib.py + tests/det_ref.py + tests/dp_ref.py): the emulated sum against a sequential fp32 loop, gloo worlds of 2 and 3
ranks for a small Qwen and a small FLUX model (identical G32 and LoRA weights on every rank, a second launch giving the same bits, the
reduced G32 equal to a one-process restatement), and the selection of the path (flag off, or ranks on several hosts: all_reduce).
GPU: the kernel against the CPU sequential sum, then two processes sharing one H100 through a gloo group and CUDA IPC training a
4-block full-width Qwen-Image-Edit model for two optimizer steps."""
import datetime
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
PATHS = (HERE, ROOT, os.path.join(ROOT, "qwen-image-finetune_b200"), os.path.join(ROOT, "tools"))
TIMEOUT = datetime.timedelta(seconds=120)  # every collective and barrier of the workers gives up after this
FLUX_YAML_R32 = 171_935_744  # flat LoRA gradient elements of FLUX-Kontext with the YAML targets at r = 32


def _paths():
    for p in PATHS:
        if p not in sys.path:
            sys.path.insert(0, p)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _special(n, w, seed):
    """fp32 [n] of rank w: normals across magnitudes plus -0.0, +0.0, denormals, +-inf and nan at fixed places."""
    g = torch.Generator().manual_seed(seed * 131 + w)
    x = torch.randn(n, generator=g) * torch.exp2(torch.randint(-30, 30, (n,), generator=g).float())
    vals = torch.tensor([-0.0, 0.0, 1e-45, -3e-42, 1.1754942e-38, float("inf"), -float("inf"), float("nan"), -1e-40, 2e-39])
    k = min(n, vals.numel())
    x[torch.randint(0, n, (k,), generator=g)] = vals[torch.randperm(vals.numel(), generator=g)[:k]]
    return x


def _sequential(srcs):
    """((+0 + s_0) + s_1) + ... with numpy float32 adds (IEEE round to nearest, denormals kept)."""
    acc = np.zeros(srcs[0].numel(), dtype=np.float32)
    for s in srcs:
        acc = np.add(acc, s.cpu().numpy().astype(np.float32), dtype=np.float32)
    return torch.from_numpy(acc)


def _same_bits(got, ref):
    """bit-identical, where a nan result only has to be some nan (qfx.h leaves its payload open)."""
    got, ref = got.cpu().reshape(-1), ref.cpu().reshape(-1)
    nan = ref.isnan()
    return bool((got.isnan() == nan).all()) and bool((got[~nan].view(torch.int32) == ref[~nan].view(torch.int32)).all())


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("world", range(1, 9))
def test_emulated_sum_is_the_sequential_loop(world):
    import dp_ref
    for n in (1, 3, 17, 4099):
        srcs = [_special(n, w, n) for w in range(world)]
        dst = torch.full((n,), 7.0)
        dp_ref.dp_reduce_det(srcs, dst)
        assert _same_bits(dst, _sequential(srcs)), (world, n)
    # in place, into one of the sources (what the reduce-scatter does)
    srcs = [_special(33, w, 5) for w in range(world)]
    ref = _sequential(srcs)
    dp_ref.dp_reduce_det(srcs, srcs[world - 1])
    assert _same_bits(srcs[world - 1], ref)
    z = torch.zeros(4)
    dp_ref.dp_reduce_det([torch.full((4,), -0.0)] * world, z)
    assert not torch.signbit(z).any(), "the sum starts from +0: -0 + ... + -0 is +0"


def _build(family):
    torch.manual_seed(7)  # identical frozen weights and adapters on every rank and in the restatement
    if family == "qwen":
        from qflux_b200.qwen_model import QwenB200Config, QwenImageB200
        m = QwenImageB200(QwenB200Config(num_layers=2, num_attention_heads=2, joint_attention_dim=128), device="cpu", _host_only=True)
        targets = ("to_q", "to_out.0", "img_mod.1", "net.2")
    else:
        from qflux_b200.flux_model import FluxB200, FluxB200Config
        m = FluxB200(FluxB200Config(num_layers=1, num_single_layers=2, attention_head_dim=128, num_attention_heads=2, joint_attention_dim=64,
                                    pooled_projection_dim=64, guidance_embeds=True), device="cpu", _host_only=True)
        targets = r".*(attn\.to_q|attn\.to_out\.0|norm1\.linear|single_transformer_blocks\.[0-9]+\.(norm\.linear|proj_mlp|proj_out)|ff\.net\.2)"
    for k, t in m.w.items():
        if k.endswith("_w") and t.ndim >= 2 and "qknorm" not in k:
            t.copy_((torch.randn(t.shape) * 0.05).bfloat16())
    m.add_adapter(4, 4, target_modules=targets, b_std=0.05)
    return m


def _step_and_batch(m, family, rank):
    from qflux_b200.train_step import FluxKontextStep, QwenImageEditStep
    g = torch.Generator().manual_seed(100 + rank)  # per-rank data
    rn = lambda *s: torch.randn(*s, generator=g).bfloat16()
    if family == "qwen":
        emb = dict(image_latents=rn(1, 16, 64), control_latents=rn(1, 16, 64), prompt_embeds=rn(1, 8, 128), img_shapes=[[(1, 4, 4), (1, 4, 4)]])
        return QwenImageEditStep(m, max_grad_norm=1.0), emb, rn(1, 16, 64), torch.tensor([0.25 + 0.125 * rank])
    emb = dict(image_latents=rn(1, 16, 64), control_latents=rn(1, 16, 64), pooled_prompt_embeds=rn(1, 64), prompt_embeds=rn(1, 8, 64),
               text_ids=torch.zeros(8, 3), image_ids=FluxKontextStep.latent_image_ids(4, 4, "cpu", 0.0),
               control_ids=FluxKontextStep.latent_image_ids(4, 4, "cpu", 1.0))
    return FluxKontextStep(m, max_grad_norm=1.0), emb, rn(1, 16, 64), torch.tensor([0.25 + 0.125 * rank]).bfloat16()


def _cpu_worker(rank, world, port, family, out):
    _paths()
    import dp_ref
    from qflux_b200 import lib
    from qflux_b200.optim import FusedLoraAdamW
    dp_ref.install(lib)
    torch.use_deterministic_algorithms(True)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=TIMEOUT)
    m = _build(family)
    step, emb, noise, t = _step_and_batch(m, family, rank)
    opt = FusedLoraAdamW(m, lr=1e-2)
    step.train_step(emb, opt, noise, t)
    res = dict(g32=m.G32.clone(), lora=torch.cat([p.detach().float().reshape(-1) for _, p in sorted(m._lora_params.items())]),
               exchange=type(m._grad_exchange).__name__)
    m.close()
    torch.save(res, f"{out}.{rank}")
    dist.destroy_process_group()


def _launch(worker, world, tmp_path, tag, *args):
    out = str(tmp_path / tag)
    mp.spawn(worker, args=(world, _free_port(), *args, out), nprocs=world, join=True)
    return [torch.load(f"{out}.{r}") for r in range(world)]


def _restated_sum(family, world):
    """One process: each rank's batch alone from a zeroed G32, then the sum in rank order from +0."""
    import dp_ref
    from qflux_b200 import lib
    restore = dp_ref.install(lib)
    torch.use_deterministic_algorithms(True)
    try:
        m = _build(family)
        grads = []
        for r in range(world):
            step, emb, noise, t = _step_and_batch(m, family, r)
            step._run(*step._prepare(emb, noise, t))
            grads.append(m.G32.clone())
    finally:
        torch.use_deterministic_algorithms(False)
        restore()
    return _sequential(grads), grads


@pytest.mark.timeout(600)
@pytest.mark.parametrize("family", ["qwen", "flux"])
@pytest.mark.parametrize("world", [2, 3])
def test_gloo_world_sums_in_rank_order(tmp_path, family, world):
    a = _launch(_cpu_worker, world, tmp_path, "a", family)
    b = _launch(_cpu_worker, world, tmp_path, "b", family)
    assert all(r["exchange"] == "GradExchange" for r in a), "the flag and one host select the fixed-order exchange"
    for r in range(world):
        assert torch.equal(a[r]["g32"].view(torch.int32), a[0]["g32"].view(torch.int32)), "every rank holds the same reduced G32"
        assert torch.equal(a[r]["lora"].view(torch.int32), a[0]["lora"].view(torch.int32)), "every rank holds the same LoRA weights"
        assert torch.equal(b[r]["g32"].view(torch.int32), a[r]["g32"].view(torch.int32)), "a second launch reproduces G32"
        assert torch.equal(b[r]["lora"].view(torch.int32), a[r]["lora"].view(torch.int32)), "a second launch reproduces the weights"
    ref, grads = _restated_sum(family, world)
    assert not torch.equal(grads[0], grads[1]), "ranks must see different batches"
    assert _same_bits(a[0]["g32"], ref), "the reduced G32 is the rank-ordered sum of the one-process gradients"


class _Calls:
    def __init__(self):
        self.all_reduce = []

    def patch(self, monkeypatch, hosts):
        monkeypatch.setattr(dist, "is_initialized", lambda: True)
        monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)
        monkeypatch.setattr(dist, "get_rank", lambda group=None: 0)
        monkeypatch.setattr(dist, "all_reduce", lambda t, *a, **k: self.all_reduce.append(t))

        def gather(out, obj, group=None):
            out[:] = [(h, obj[1]) for h in hosts]
        monkeypatch.setattr(dist, "all_gather_object", gather)


@pytest.mark.parametrize("flag,hosts", [(False, ("a", "a")), (True, ("a", "b"))])
def test_nccl_all_reduce_stays_where_the_exchange_does_not_apply(monkeypatch, flag, hosts):
    """Flag off: the exchange is not even consulted.  Flag on with ranks on two hosts: it declines and NCCL's all-reduce runs."""
    import dp_ref
    from qflux_b200 import lib
    from qflux_b200.optim import FusedLoraAdamW
    from qflux_b200.train_step import _sync_and_step
    restore = dp_ref.install(lib)
    was = torch.are_deterministic_algorithms_enabled()
    try:
        m = _build("qwen")
        opt = FusedLoraAdamW(m, lr=1e-2)
        m.G32.normal_()
        g32 = m.G32
        calls = _Calls()
        calls.patch(monkeypatch, hosts)
        torch.use_deterministic_algorithms(flag)
        _sync_and_step(m, opt, 1.0)
        assert len(calls.all_reduce) == 1 and calls.all_reduce[0] is g32
        assert m._grad_exchange is (False if flag else None)
        assert opt.grad_divisor == 2
    finally:
        torch.use_deterministic_algorithms(was)
        restore()


def test_graph_is_recorded_again_after_the_accumulator_moves(monkeypatch):
    """A CUDA graph bakes in G32's address: once the exchange moves G32 into peer memory, the cached graph is recorded again."""
    import contextlib
    from qflux_b200.mmdit_base import GraphCache

    class G:
        def replay(self):
            pass

    class M:
        dev, _sharded, _fwd_gen = torch.device("cuda"), None, 0

        def __init__(self):
            self._ws, self._ws_key, self.G32 = {}, "k", torch.zeros(4)
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)
    monkeypatch.setattr(torch.cuda, "CUDAGraph", G)
    records = []
    monkeypatch.setattr(torch.cuda, "graph", lambda g: (records.append(g), contextlib.nullcontext())[1])
    cache, m = GraphCache(4, "test"), M()
    for _ in range(3):
        cache.run(m, lambda x: x, (torch.ones(1),))
    assert len(records) == 1
    m.G32 = torch.zeros(4)
    cache.run(m, lambda x: x, (torch.ones(1),))
    assert len(records) == 2


def test_kernel_refuses_bad_arguments_without_gpu():
    import ctypes as C
    from qflux_b200 import lib
    L = lib._lib
    buf = torch.zeros(64)
    p = buf.data_ptr() + (-buf.data_ptr()) % 16
    arr = lambda *ps: (C.c_void_p * len(ps))(*ps)
    cases = [(arr(p), 0, p, 4, "bad arguments"), (arr(*[p] * 9), 9, p + 256, 4, "bad arguments"), (arr(p), 1, p, -1, "bad arguments"),
             (arr(p), 1, p + 2, 4, "dst must be 4-byte aligned"), (arr(0), 1, p, 4, "src[0] is NULL"),
             (arr(p + 4), 1, p, 4, "src[0] overlaps dst")]
    for src, nsrc, dst, n, msg in cases:
        rc = L.qfx_dp_reduce_det(src, nsrc, C.c_void_p(dst), n, None)
        assert rc == -1 and msg in L.qfx_last_error().decode(), (nsrc, n, L.qfx_last_error())


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3, 8])
def test_kernel_is_the_sequential_sum(world):
    from qflux_b200 import lib
    for n in (1, 3, 4099, FLUX_YAML_R32):
        srcs = [_special(n, w, n % 1000) for w in range(world)]
        ref = _sequential(srcs)
        for off in (0, 1, 3):  # slice offsets in elements: 16-byte aligned, then not
            dev = [torch.empty(n + 4, device="cuda") for _ in range(world)]
            for d, s in zip(dev, srcs):
                d[off: off + n] = s.cuda()
            dst = torch.full((n + 4,), 7.0, device="cuda")
            lib.dp_reduce_det([d[off: off + n] for d in dev], dst[off: off + n])
            assert _same_bits(dst[off: off + n], ref), (world, n, off)
            assert (dst[:off] == 7).all() and (dst[off + n:] == 7).all(), "nothing outside dst is written"
            if n > 5000:
                lib.dp_reduce_det([d[off: off + n] for d in dev], dev[1][off: off + n])  # in place into a source
                assert _same_bits(dev[1][off: off + n], ref), (world, n, off, "in place")
                # sources at different offsets from dst: the scalar path
                lib.dp_reduce_det([dev[0][1: 1 + n]] + [d[off: off + n] for d in dev[1:]], dst[:n])
                ref2 = _sequential([dev[0][1: 1 + n].cpu()] + [d[off: off + n].cpu() for d in dev[1:]])
                assert _same_bits(dst[:n], ref2), (world, n, off, "mixed alignment")
            del dev, dst
        torch.cuda.empty_cache()


def _qwen_full_width(opt_kind):
    _paths()
    import bench
    import fp8_check
    from qflux_b200.optim import FusedLoraAdam8bit, FusedLoraAdamW
    cfg = dict(bench.CONFIGS["qwen_edit"], B=1, blocks=4)
    torch.manual_seed(0)
    m = fp8_check.build("qwen", cfg, fp8=False)
    opt = FusedLoraAdamW(m, lr=1e-3) if opt_kind == "adamw" else FusedLoraAdam8bit(m, lr=1e-3)
    return m, cfg, opt


def _qwen_batch(cfg, rank):
    import bench
    torch.manual_seed(1000 + rank)
    host = bench.make_batch(cfg, "qwen_edit", host=False)
    bf = ("image_latents", "control_latents", "prompt_embeds")
    b = {k: (v.cuda().bfloat16() if k in bf else v) for k, v in host.items()}
    g = torch.Generator(device="cuda").manual_seed(2000 + rank)
    return b, torch.randn(b["image_latents"].shape, device="cuda", generator=g).bfloat16(), torch.tensor([0.25 + 0.5 * rank])


def _gpu_worker(rank, world, port, opt_kind, out):
    _paths()
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.cuda.set_device(0)  # both ranks share the one GPU
    torch.use_deterministic_algorithms(True)
    from qflux_b200.train_step import QwenImageEditStep
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=TIMEOUT)
    try:
        m, cfg, opt = _qwen_full_width(opt_kind)
        batch, noise, u = _qwen_batch(cfg, rank)
        step = QwenImageEditStep(m, "mse", max_grad_norm=1.0)
        losses = [step.train_step(batch, opt, noise, u).clone()]
        g32 = m.G32.cpu()
        losses.append(step.train_step(batch, opt, noise, u).clone())
        lora = torch.cat([p.detach().float().reshape(-1) for _, p in sorted(m._lora_params.items())]).cpu()
        res = dict(g32=g32, lora=lora, losses=[float(x) for x in losses], exchange=type(m._grad_exchange).__name__,
                   graphs=step._graphs.captured())
        m.close()
        torch.save(res, f"{out}.{rank}")
    finally:
        dist.destroy_process_group()


def _gpu_restated_sum(opt_kind, world):
    from qflux_b200.train_step import QwenImageEditStep
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        m, cfg, _ = _qwen_full_width(opt_kind)
        step = QwenImageEditStep(m, "mse", max_grad_norm=1.0)
        grads = []
        for r in range(world):
            batch, noise, u = _qwen_batch(cfg, r)
            step._run(*step._prepare(batch, noise, u))
            grads.append(m.G32.cpu())
        del m, step
    finally:
        torch.use_deterministic_algorithms(was)
        torch.cuda.empty_cache()
    return _sequential(grads), grads


@pytest.mark.gpu
@pytest.mark.timeout(1800)
@pytest.mark.parametrize("opt_kind,launches", [("adamw", 2), ("adam8bit", 1)])
def test_two_processes_on_one_gpu(tmp_path, opt_kind, launches):
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    runs = [_launch(_gpu_worker, 2, tmp_path, f"run{i}", opt_kind) for i in range(launches)]
    a = runs[0]
    assert all(r["exchange"] == "GradExchange" for r in a)
    assert a[0]["graphs"] >= 1, "the second step replays a graph recorded on the moved accumulator"
    assert torch.equal(a[0]["lora"].view(torch.int32), a[1]["lora"].view(torch.int32)), "both ranks hold the same LoRA weights"
    assert torch.equal(a[0]["g32"].view(torch.int32), a[1]["g32"].view(torch.int32))
    for b in runs[1:]:
        for r in range(2):
            assert torch.equal(b[r]["lora"].view(torch.int32), a[r]["lora"].view(torch.int32)), "a second launch reproduces the weights"
            assert b[r]["losses"] == a[r]["losses"]
    ref, grads = _gpu_restated_sum(opt_kind, 2)
    assert not torch.equal(grads[0], grads[1])
    assert _same_bits(a[0]["g32"], ref), "step 1's reduced G32 is the rank-ordered sum of the one-process gradients"
