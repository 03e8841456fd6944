"""Sharded optimizer state (optim.py shard_state=True, sharding.SlicePlan / ShardExchange, qfx.h "slice forms"): every data-parallel rank
keeps and steps the state of its slice of the flat LoRA gradient, then the ranks all-gather the updated LoRA weights.

CPU (emulated kernels: tests/emu_lib.py, det_ref.py, dp_ref.py, prodigy_ref.py, adam8bit_ref.py and shard_ref.py): gloo worlds of 2 and
3 ranks for a small Qwen and a small FLUX model and each fused optimizer, against one replicated optimizer stepped on the rank-ordered
sum of the same per-rank gradients — bit for bit when the clip is inactive, to the stated bounds when it clips; the slice plan's
properties; gradient accumulation through train_step; run-to-run repeats; checkpoints across sharded / replicated runs and world sizes;
the refusals.  GPU: every new kernel per element at the FLUX-YAML r = 32 tables, and two processes sharing one H100."""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
PATHS = (HERE, ROOT, os.path.join(ROOT, "qwen-image-finetune_b200"), os.path.join(ROOT, "tools"))
for _p in PATHS:
    if _p not in sys.path:
        sys.path.insert(0, _p)

from test_dp_determinism import TIMEOUT, _build, _free_port, _paths, _sequential, _step_and_batch  # noqa: E402

NO_CLIP, CLIP = 1e9, 1e-3


def _make(kind, m, shard_state):
    from qflux_b200.optim import FusedLoraAdam8bit, FusedLoraAdamW, FusedLoraProdigy
    if kind == "adamw":
        return FusedLoraAdamW(m, lr=1e-2, shard_state=shard_state)
    if kind == "prodigy":
        return FusedLoraProdigy(m, lr=1.0, d0=1e-4, shard_state=shard_state)
    return FusedLoraAdam8bit(m, lr=1e-2, min_8bit_size=512, shard_state=shard_state)


def _grad(n, rank, step):
    g = torch.Generator().manual_seed(1000 * step + rank)
    return torch.randn(n, generator=g) * 0.01


def _lora(m):
    return torch.cat([p.detach().reshape(-1) for _, p in sorted(m._lora_params.items())])


def _set_lora(m, flat):
    o = 0
    for _, p in sorted(m._lora_params.items()):
        p.data.copy_(flat[o: o + p.numel()].view(p.shape))
        o += p.numel()


def _worker(rank, world, port, family, kind, clip, flag, steps, init, out):
    _paths()
    import shard_ref
    from qflux_b200 import lib
    from qflux_b200.train_step import _sync_and_step
    shard_ref.install(lib)
    torch.use_deterministic_algorithms(flag)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=TIMEOUT)
    m = _build(family)
    opt = _make(kind, m, True)
    first = 0
    if init is not None:
        ck = torch.load(init)
        _set_lora(m, ck["lora"])
        opt.load_state_dict(ck["sd"])
        first = ck["steps"]
    for s in range(first, first + steps):
        m.G32.copy_(_grad(m.G32.numel(), rank, s))
        _sync_and_step(m, opt, clip)
    res = dict(lora=_lora(m), sd=opt.state_dict(), norm=opt.grad_norm_sq.clone(), steps=first + steps,
               state_numel=sum(getattr(opt, k).numel() for k in ("exp_avg", "state1") if hasattr(opt, k)))
    m.close()
    torch.save(res, f"{out}.{rank}")
    dist.destroy_process_group()


def _launch(tmp_path, tag, world, *args):
    out = str(tmp_path / tag)
    mp.spawn(_worker, args=(world, _free_port(), *args, out), nprocs=world, join=True)
    return [torch.load(f"{out}.{r}") for r in range(world)]


def _replicated(family, kind, clip, world, steps, init=None):
    """One process, one replicated optimizer: each step's gradient is the rank-ordered sum of the ranks' gradients."""
    import shard_ref
    from qflux_b200 import lib
    restore = shard_ref.install(lib)
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        m = _build(family)
        opt = _make(kind, m, False)
        first = 0
        if init is not None:
            _set_lora(m, init["lora"])
            opt.load_state_dict(init["sd"])
            first = init["steps"]
        for s in range(first, first + steps):
            m.G32.copy_(_sequential([_grad(m.G32.numel(), r, s) for r in range(world)]))
            opt.max_grad_norm = clip
            opt.step(grad_divisor=world)
        return dict(lora=_lora(m), sd=opt.state_dict(), norm=opt.grad_norm_sq.clone(), steps=first + steps)
    finally:
        torch.use_deterministic_algorithms(was)
        restore()


def _bits(a, b):
    if torch.is_tensor(a):
        return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.reshape(-1).view(torch.uint8), b.reshape(-1).view(torch.uint8))
    return a == b


def _same_state(sd, ref):
    f, g = sd["fused"], ref["fused"]
    assert f.keys() == g.keys()
    for k in f:
        assert _bits(f[k], g[k]), k
    assert sd["param_groups"] == ref["param_groups"]


def _within_one_ulp(a, b):
    """bf16 tensors at most one unit in the last place apart."""
    d = (a.view(torch.int16).int() - b.view(torch.int16).int()).abs()
    return bool(((d <= 1) | (a == b)).all())


# ------------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.timeout(900)
@pytest.mark.parametrize("kind", ["adamw", "prodigy", "adam8bit"])
@pytest.mark.parametrize("family", ["qwen", "flux"])
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_equals_replicated(tmp_path, world, family, kind):
    got = _launch(tmp_path, "a", world, family, kind, NO_CLIP, True, 3, None)
    ref = _replicated(family, kind, NO_CLIP, world, 3)
    assert not torch.equal(ref["lora"], _replicated(family, kind, NO_CLIP, world, 0)["lora"]), "the steps change the weights"
    for r in range(world):
        assert _bits(got[r]["lora"], ref["lora"]), f"rank {r}: the LoRA weights are the replicated optimizer's"
        _same_state(got[r]["sd"], ref["sd"])
        assert torch.allclose(got[r]["norm"], ref["norm"], rtol=1e-6, atol=0)
    n = ref["sd"]["fused"]["exp_avg" if kind != "adam8bit" else "state1"].numel()
    assert sum(g["state_numel"] for g in got) == n, "the slices' state adds up to the replicated state"


@pytest.mark.timeout(900)
@pytest.mark.parametrize("kind", ["adamw", "prodigy", "adam8bit"])
def test_clipped_step_stays_within_one_ulp(tmp_path, kind):
    got = _launch(tmp_path, "a", 2, "flux", kind, CLIP, True, 3, None)
    ref = _replicated("flux", kind, CLIP, 2, 3)
    for g in got:
        assert torch.allclose(g["norm"], ref["norm"], rtol=1e-6, atol=0)
        assert _within_one_ulp(g["lora"], ref["lora"])
    assert _bits(got[0]["lora"], got[1]["lora"]), "every rank holds the same weights"


@pytest.mark.timeout(900)
@pytest.mark.parametrize("flag", [True, False])
def test_run_to_run_is_bit_identical(tmp_path, flag):
    a = _launch(tmp_path, "a", 3, "qwen", "prodigy", CLIP, flag, 2, None)
    b = _launch(tmp_path, "b", 3, "qwen", "prodigy", CLIP, flag, 2, None)
    for r in range(3):
        assert _bits(a[r]["lora"], b[r]["lora"]) and _bits(a[r]["norm"], b[r]["norm"])
        _same_state(a[r]["sd"], b[r]["sd"])


@pytest.mark.timeout(900)
@pytest.mark.parametrize("kind", ["adamw", "prodigy", "adam8bit"])
def test_checkpoints_move_between_world_sizes(tmp_path, kind):
    two = _launch(tmp_path, "w2", 2, "flux", kind, NO_CLIP, True, 2, None)
    path = str(tmp_path / "ck.pt")
    torch.save(two[0], path)
    ref = _replicated("flux", kind, NO_CLIP, 2, 2)
    assert _bits(two[0]["lora"], ref["lora"])
    # world 3 continues the world-2 checkpoint; its gradients are the rank sums of three ranks from here on
    three = _launch(tmp_path, "w3", 3, "flux", kind, NO_CLIP, True, 1, path)
    ref3 = _replicated("flux", kind, NO_CLIP, 3, 1, init=ref)
    rep = _replicated("flux", kind, NO_CLIP, 3, 1, init=two[0])  # the sharded checkpoint loads into a replicated optimizer
    for r in range(3):
        assert _bits(three[r]["lora"], ref3["lora"])
        _same_state(three[r]["sd"], ref3["sd"])
    assert _bits(rep["lora"], ref3["lora"])
    _same_state(rep["sd"], ref3["sd"])


def test_slice_plan_properties():
    from qflux_b200 import lib
    from qflux_b200.sharding import SlicePlan
    sizes = [5000, 64, 4096, 12288 + 3, 1, 8192, 300, 4097]
    members, off = [], 0
    for n in sizes:
        members.append((torch.zeros(1, n), off))
        off += n + 5  # gaps between tensors
    for world in range(2, 9):
        plan = SlicePlan(members, off, world)
        covered = [c for c0, c1 in plan.chunk_ranges for c in range(c0, c1)]
        assert covered == list(range(len(plan.chunks))), "contiguous, disjoint and covering every chunk"
        assert plan.bounds[0][0] == 0 and plan.bounds[-1][1] == off
        assert all(plan.bounds[q][1] == plan.bounds[q + 1][0] for q in range(world - 1)), "the slices partition G32"
        mean = sum(sizes) / world
        assert all(abs(e - mean) <= lib.ADAMW_CHUNK for e in plan.elements), (world, plan.elements)
        for q, (c0, c1) in enumerate(plan.chunk_ranges):
            for i, e, g, n in plan.chunks[c0:c1]:
                assert e % lib.ADAM8BIT_BLOCK == 0 and plan.bounds[q][0] <= g and g + n <= plan.bounds[q][1], "no 8-bit block is cut"
            for i, e0, e1 in plan.pieces(q):
                assert e0 % lib.ADAMW_CHUNK == 0 and (e1 % lib.ADAMW_CHUNK == 0 or e1 == sizes[i])
    with pytest.raises(ValueError):
        SlicePlan([(torch.zeros(1, 8), 4), (torch.zeros(1, 8), 0)], 16, 2)


@pytest.mark.timeout(900)
def test_gradient_accumulation_through_train_step(tmp_path):
    out = str(tmp_path / "acc")
    mp.spawn(_accum_worker, args=(2, _free_port(), out), nprocs=2, join=True)
    got = [torch.load(f"{out}.{r}") for r in range(2)]
    import shard_ref
    from qflux_b200 import lib
    restore = shard_ref.install(lib)
    torch.use_deterministic_algorithms(True)
    try:
        m = _build("qwen")
        grads = []
        for r in range(2):
            for micro in range(2):
                step, emb, noise, t = _step_and_batch(m, "qwen", 2 * r + micro)
                step._accumulating = micro > 0
                step._run(*step._prepare(emb, noise, t))
            grads.append(m.G32.clone())
        opt = _make("adamw", m, False)
        m.G32.copy_(_sequential(grads))
        opt.max_grad_norm = NO_CLIP
        opt.step(grad_divisor=4)
        ref = _lora(m)
    finally:
        torch.use_deterministic_algorithms(False)
        restore()
    for g in got:
        assert _bits(g, ref)


def _accum_worker(rank, world, port, out):
    _paths()
    import shard_ref
    from qflux_b200 import lib
    from qflux_b200.train_step import QwenImageEditStep
    shard_ref.install(lib)
    torch.use_deterministic_algorithms(True)
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=TIMEOUT)
    m = _build("qwen")
    opt = _make("adamw", m, True)
    step = QwenImageEditStep(m, max_grad_norm=NO_CLIP, gradient_accumulation_steps=2)
    for micro in range(2):
        _, emb, noise, t = _step_and_batch(m, "qwen", 2 * rank + micro)
        step.train_step(emb, opt, noise, t)
    torch.save(_lora(m), f"{out}.{rank}")
    m.close()
    dist.destroy_process_group()


def test_refusals(monkeypatch):
    import emu_lib
    from qflux_b200 import lib
    restore = emu_lib.install(lib)
    try:
        m = _build("qwen")
        for kind in ("adamw", "prodigy", "adam8bit"):
            with pytest.raises(lib.QfxError, match="initialised torch.distributed"):
                _make(kind, m, True)
        monkeypatch.setattr(dist, "is_initialized", lambda: True)
        monkeypatch.setattr(dist, "get_world_size", lambda group=None: 1)
        for kind in ("adamw", "prodigy", "adam8bit"):
            with pytest.raises(lib.QfxError, match="2 or more ranks, got 1"):
                _make(kind, m, True)
    finally:
        restore()


def test_entry_points_refuse_bad_arguments_without_gpu():
    import ctypes as C
    from qflux_b200 import lib
    L, vp = lib._lib, C.c_void_p
    buf = torch.zeros(1024)
    p = vp(buf.data_ptr())
    f = C.c_float
    cases = [
        ("qfx_sumsq_det", lambda: L.qfx_sumsq_det(vp(0), C.c_int64(4), f(1), p, p, C.c_int64(4096), None), "bad arguments"),
        ("qfx_sumsq_det", lambda: L.qfx_sumsq_det(p, C.c_int64(4), f(1), p, p, C.c_int64(8), None), "needs 592"),
        ("qfx_fused_adamw_slice", lambda: lib._adamw_slice(p, p, 1, p, 100, 90, 20, p, p, p, 1, 1, 1, 0.9, 0.99, 1e-8, 0, 1, None),
         "bad arguments"),
        ("qfx_fused_adamw_slice", lambda: lib._adamw_slice(p, p, 1, p, 100, 0, 10, vp(0), p, p, 1, 1, 1, 0.9, 0.99, 1e-8, 0, 1, None),
         "bad arguments"),
        ("qfx_fused_adam8bit_slice", lambda: lib._adam8bit_slice(p, p, 1, p, p, 100, -1, 10, p, p, p, p, p, p, p, p, p, 1, 1, 1, 0.9,
                                                                 0.99, 1e-8, 0, 1, 0, None), "bad arguments"),
        ("qfx_fused_adam8bit_slice", lambda: lib._adam8bit_slice(p, p, 1, p, p, 100, 0, 10, p, p, p, p, p, p, p, p, p, 1, 1, -1, 0.9,
                                                                 0.99, 1e-8, 0, 1, 0, None), "lr >= 0"),
        ("qfx_prodigy_slice_partials", lambda: lib._prodigy_a(p, p, 3, 2, p, 100, 0, 10, p, p, p, p, p, p, p, 4, 1, 1, 1, .9, .99, .99,
                                                              0, 1, 0, 0, 1e-6, None), "bad arguments"),
        ("qfx_prodigy_slice_partials", lambda: lib._prodigy_a(p, p, 1, 0, p, 100, 0, 10, p, p, p, p, p, p, p, 4, 1, 1, 0, .9, .99, .99,
                                                              0, 1, 0, 0, 1e-6, None), "lr > 0"),
        ("qfx_prodigy_slice_update", lambda: lib._prodigy_b(p, p, 1, 100, 0, 10, p, p, p, p, 0, 1, .9, .99, .99, 1e-8, 0, 1, 0, 1e-6, 1,
                                                            1e30, None), "bad arguments"),
        ("qfx_lora_pack", lambda: lib._pack(p, p, 1, 10, 5, p, None), "bad arguments"),
        ("qfx_lora_unpack", lambda: lib._unpack(p, p, 1, 0, 5, vp(buf.data_ptr() + 1), None), "2-byte aligned"),
    ]
    for name, call, msg in cases:
        rc = call()
        assert rc == -1 and msg in L.qfx_last_error().decode(), (name, L.qfx_last_error())


# ------------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
@pytest.mark.timeout(900)
@pytest.mark.parametrize("case", ["pack", "sumsq", "adamw", "adam8bit", "prodigy"])
def test_kernels_per_element(case):
    import subprocess
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "sharded_optim_check.py"), case], capture_output=True, text=True)
    print(r.stdout, r.stderr[-4000:])
    assert r.returncode == 0, r.stdout + r.stderr[-4000:]


def _gpu_model(kind, shard_state):
    import bench
    import fp8_check
    cfg = dict(bench.CONFIGS["qwen_edit"], B=1, blocks=4)
    torch.manual_seed(0)
    m = fp8_check.build("qwen", cfg, fp8=False)
    return m, cfg, _make(kind, m, shard_state)


def _state_bytes(opt):
    keys = ("exp_avg", "exp_avg_sq", "s", "p0", "state1", "state2", "absmax1", "absmax2", "s1_32", "s2_32")
    return sum(getattr(opt, k).numel() * getattr(opt, k).element_size() for k in keys if hasattr(opt, k))


def _two_gpu_worker(rank, world, port, kind, flag, out):
    _paths()
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.cuda.set_device(0)  # both ranks share the one GPU
    torch.use_deterministic_algorithms(flag)
    from test_dp_determinism import _qwen_batch
    from qflux_b200.train_step import QwenImageEditStep
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=TIMEOUT)
    try:
        m, cfg, opt = _gpu_model(kind, True)
        step = QwenImageEditStep(m, "mse", max_grad_norm=NO_CLIP)
        for s in range(2):
            batch, noise, u = _qwen_batch(cfg, 2 * s + rank)
            step.train_step(batch, opt, noise, u)
        res = dict(lora=_lora(m).cpu(), state_bytes=_state_bytes(opt), exchange=type(m._grad_exchange).__name__,
                   n_grad=m.G32.numel(), elements=opt._plan.elements[rank])
        m.close()
        torch.save(res, f"{out}.{rank}")
    finally:
        dist.destroy_process_group()


def _gpu_replicated(kind):
    from test_dp_determinism import _qwen_batch
    from qflux_b200 import lib
    from qflux_b200.train_step import QwenImageEditStep
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        m, cfg, opt = _gpu_model(kind, False)
        step = QwenImageEditStep(m, "mse", max_grad_norm=NO_CLIP)
        for s in range(2):
            grads = []
            for r in range(2):
                batch, noise, u = _qwen_batch(cfg, 2 * s + r)
                step._run(*step._prepare(batch, noise, u))
                grads.append(m.G32.clone())
            lib.dp_reduce_det(grads, m.G32)
            opt.max_grad_norm = NO_CLIP
            opt.step(grad_divisor=2)
        res = dict(lora=_lora(m).cpu(), state_bytes=_state_bytes(opt))
        del m, opt, step
        return res
    finally:
        torch.use_deterministic_algorithms(was)
        torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.timeout(1800)
@pytest.mark.parametrize("kind", ["adamw", "prodigy"])
def test_two_processes_on_one_gpu(tmp_path, kind):
    """Flag on: the peer-memory reduce-scatter, bit-equal to the replicated optimizer.  Flag off: the collectives path (gloo here:
    all_gather and the rank-ordered sum; the backward kernels use atomics, so the weights are compared to a bound)."""
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    ref = _gpu_replicated(kind)
    for flag in (True, False):
        out = str(tmp_path / f"f{int(flag)}")
        mp.spawn(_two_gpu_worker, args=(2, _free_port(), kind, flag, out), nprocs=2, join=True)
        got = [torch.load(f"{out}.{r}") for r in range(2)]
        assert _bits(got[0]["lora"], got[1]["lora"]), "both ranks hold the same weights"
        if flag:
            assert got[0]["exchange"] == "GradExchange"
            assert _bits(got[0]["lora"], ref["lora"]), "the sharded run equals the replicated run bit for bit"
        else:
            rel = float((got[0]["lora"].float() - ref["lora"].float()).norm() / ref["lora"].float().norm())
            assert rel < 1e-2, rel
        per_elt = ref["state_bytes"] / got[0]["n_grad"]
        for r in range(2):
            assert abs(got[r]["state_bytes"] - ref["state_bytes"] / 2) <= per_elt * 4096 + 64, (got[r]["state_bytes"], ref["state_bytes"])
