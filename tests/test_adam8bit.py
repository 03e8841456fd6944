"""FusedLoraAdam8bit: the configs' bitsandbytes.optim.Adam8bit as fused kernels over the flat LoRA gradient (qfx.h qfx_fused_adam8bit).

CPU (kernels emulated by tests/emu_lib.py + tests/adam8bit_ref.py): the dynamic maps, 20 steps of a cosine warm-up from lr 0 against the
restatement of bitsandbytes' Adam8bit (tests/adam8bit_ref.py) bit for bit, the boundary shapes, the lr-0 step, a state_dict round trip,
refused arguments, the C argument checks, a gloo world-2 run and a gradient-accumulation-2 train_step.
GPU (tools/adam8bit_check.py, one subprocess per case): the kernel at full FLUX-YAML size checked step by step against the restatement
started from the kernel's own state, the boundary shapes on the device, bitwise repeats, and three `train_step`s per model."""
import copy
import ctypes as C
import json
import math
import os
import socket
import subprocess
import sys
from importlib.util import find_spec

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tools"))
CHECK = os.path.join(ROOT, "tools", "adam8bit_check.py")

CONFIG_ARGS = dict(lr=1e-4, betas=[0.9, 0.999])  # the eight Adam8bit configs' init_args


@pytest.fixture()
def emu():
    import adam8bit_ref
    from qflux_b200 import lib
    restore = adam8bit_ref.install(lib)
    yield lib
    restore()


def _model(seed=7, r=8):
    """r = 8 on a 256-wide model: the attention factors (2048 elements) take the fp32 path, the MLP's [1024, 8] / [8, 1024] the 8-bit one."""
    from qflux_b200.qwen_model import QwenB200Config, QwenImageB200
    torch.manual_seed(seed)
    m = QwenImageB200(QwenB200Config(num_layers=1, num_attention_heads=2, joint_attention_dim=128), device="cpu", _host_only=True)
    m.add_adapter(r, r, target_modules=["to_q", "to_k", "to_v", "to_out.0", "img_mlp.net.0.proj", "img_mlp.net.2"], b_std=0.05)
    return m


def cosine_warmup(opt, warmup=5, total=20):
    """diffusers.optimization.get_cosine_schedule_with_warmup (num_cycles = 0.5), the configs' `scheduler_type: cosine`"""
    def f(step):
        if step < warmup:
            return step / max(1, warmup)
        prog = (step - warmup) / max(1, total - warmup)
        return max(0.0, 0.5 * (1.0 + math.cos(math.pi * 0.5 * 2.0 * prog)))
    return torch.optim.lr_scheduler.LambdaLR(opt, f)


def _grads(m, t):
    g = torch.Generator().manual_seed(1000 + t)
    return torch.randn(m.G32.shape, generator=g) * 0.05


def _restated_step(ref_opt, ps, m, G, pre_scale, max_norm):
    """Feed the restatement the flat gradient the way the emulated kernel sees it: G * pre_scale, times the fp32 clip coefficient."""
    import adam8bit_ref
    g = G * np.float32(pre_scale)
    g = g * torch.tensor(adam8bit_ref.clip_coef(g, max_norm), dtype=torch.float32)
    for (p, off), q in zip(_members(m), ps):
        q.grad_dtype = None  # an fp32 gradient on a bf16 parameter
        q.grad = g[off: off + p.numel()].view(p.shape).clone()
    ref_opt.step()


def _members(m):
    out = []
    for full, pA, pB, ga, gb, d_in, d_out in m._all_members():
        out += [(pA, ga), (pB, gb)]
    return out


@pytest.mark.parametrize("kw", [CONFIG_ARGS, dict(), dict(weight_decay=0.01)], ids=["configs", "defaults", "weight_decay"])
def test_matches_restated_adam8bit_over_cosine_warmup(emu, kw):
    """20 steps of a cosine warm-up starting at lr 0, with the clip active: every LoRA parameter, code, absmax and fp32 state of
    FusedLoraAdam8bit equals the restatement's, bit for bit; both paths (8-bit and fp32) are exercised."""
    import adam8bit_ref
    from qflux_b200.optim import FusedLoraAdam8bit
    m = _model()
    ps = [torch.nn.Parameter(p.detach().clone()) for p, _ in _members(m)]
    ref = adam8bit_ref.Adam8bit(ps, **kw)
    opt = FusedLoraAdam8bit(m, **kw, max_grad_norm=1.0)
    sch, sch_r = cosine_warmup(opt), cosine_warmup(ref)
    sizes = [p.numel() for p in ps]
    assert min(sizes) < 4096 <= max(sizes), "both state paths must be covered"
    for t in range(20):
        m.G32.copy_(_grads(m, t))
        _restated_step(ref, ps, m, m.G32, 1.0, 1.0)
        opt.step()
        sch.step()
        sch_r.step()
    offsets = opt.state_offsets.tolist()
    for (p, off), q, so in zip(_members(m), ps, offsets):
        n, st = p.numel(), ref.state[q]
        assert st["step"] == opt.step_count == 20
        assert torch.equal(p.detach(), q.detach())
        if "absmax1" in st:
            nb = st["absmax1"].numel()
            assert torch.equal(opt.state1[off: off + n], st["state1"]) and torch.equal(opt.state2[off: off + n], st["state2"])
            assert torch.equal(opt.absmax1[so: so + nb], st["absmax1"]) and torch.equal(opt.absmax2[so: so + nb], st["absmax2"])
            assert st["absmax1"].gt(0).all() and st["absmax2"].gt(0).all()
        else:
            assert torch.equal(opt.s1_32[so: so + n], st["state1"]) and torch.equal(opt.s2_32[so: so + n], st["state2"])


def test_dynamic_maps():
    import adam8bit_ref
    from qflux_b200 import lib
    for signed, zero in ((True, 127), (False, 0)):
        q = adam8bit_ref.create_dynamic_map(signed)
        assert q.shape == (256,) and q.dtype == torch.float32
        assert torch.all(q[1:] > q[:-1]), "sorted, no repeated entries"
        assert q[zero] == 0 and q[255] == 1.0
        assert torch.equal(lib.dynamic_map(signed), q)
    assert abs(float(adam8bit_ref.create_dynamic_map(True)[0]) + 0.993) < 1e-3


@pytest.mark.skipif(find_spec("bitsandbytes") is None, reason="bitsandbytes is not installed")
def test_dynamic_maps_against_bitsandbytes():
    import bitsandbytes.functional as F
    from qflux_b200 import lib
    for signed in (True, False):
        assert torch.equal(lib.dynamic_map(signed), F.create_dynamic_map(signed=signed).float().cpu())


def test_quantize_rule():
    """nearest entry, ties to the lower code; the sign rule moves tiny negative first states to the smallest negative code; a zero
    absmax stores the zero codes"""
    import adam8bit_ref as ar
    q1, q2 = ar.create_dynamic_map(True), ar.create_dynamic_map(False)
    x = torch.tensor([q1[200], q1[200] * 0.5 + q1[201] * 0.5, 1.0, -1.0, 0.0])
    assert ar.quantize(q1, x).tolist() == [200, 200, 255, 0, 127]
    s1 = torch.tensor([-1e-9, 1e-9, 0.5, 0.0] + [0.0] * 252)
    s2 = torch.tensor([1e-9, 0.0, 0.5, 0.0] + [0.0] * 252)
    c1, c2 = ar.quantize_states(s1, s2, ar.block_absmax(s1), ar.block_absmax(s2), q1, q2)
    assert c1[:4].tolist() == [126, 127, 255, 127] and c2[:4].tolist() == [0, 0, 255, 0]
    c1, c2 = ar.quantize_states(torch.zeros(300), torch.zeros(300), torch.zeros(2), torch.zeros(2), q1, q2)
    assert c1.eq(ar.CODE1_ZERO).all() and c2.eq(ar.CODE2_ZERO).all()


def test_boundary_shapes(emu):
    """numel 4095 (fp32 path) and 4096 (8-bit), 5000 elements (partial last block), a row-strided B view whose padding stays zero, an
    all-zero-gradient block: the same case tools/adam8bit_check.py runs on the device, here on the emulation."""
    import adam8bit_check
    res = adam8bit_check.kernel_small_and_partial("cpu")
    assert not res["fail"], res


def test_layout():
    from qflux_b200 import lib
    ps = [torch.zeros(s) for s in ((4095,), (4096,), (5000,), (10,))]
    offsets, n_absmax, n_small = lib.adam8bit_layout([(p, 0) for p in ps], 4096)
    assert offsets == [0, 0, 16, 4095] and n_absmax == 16 + 20 and n_small == 4105


def test_lr_zero_step_moves_states_not_parameters(emu):
    from qflux_b200.optim import FusedLoraAdam8bit
    m = _model()
    opt = FusedLoraAdam8bit(m, **CONFIG_ARGS)
    before = [p.detach().clone() for p in m.parameters()]
    opt.param_groups[0]["lr"] = 0.0
    m.G32.copy_(_grads(m, 0))
    opt.step()
    assert opt.step_count == 1
    assert all(torch.equal(a, b) for a, b in zip(before, m.parameters()))
    assert opt.state1.any() and opt.state2.any() and opt.absmax1.gt(0).all() and opt.absmax2.gt(0).all() and opt.s1_32.any()


def test_state_dict_round_trip_continues_bit_for_bit(emu):
    from qflux_b200.optim import FusedLoraAdam8bit
    m = _model()
    opt = FusedLoraAdam8bit(m, **CONFIG_ARGS)
    sch = cosine_warmup(opt)

    def run(o, s, model, t0, t1):
        for t in range(t0, t1):
            model.G32.copy_(_grads(model, t))
            o.step()
            s.step()
    run(opt, sch, m, 0, 8)
    saved_opt, saved_sch = copy.deepcopy(opt.state_dict()), copy.deepcopy(sch.state_dict())
    saved_params = {n: p.detach().clone() for n, p in m._lora_params.items()}
    run(opt, sch, m, 8, 14)
    m2 = _model()
    with torch.no_grad():
        for n, p in m2._lora_params.items():
            p.copy_(saved_params[n])
    opt2 = FusedLoraAdam8bit(m2, **CONFIG_ARGS)
    sch2 = cosine_warmup(opt2)
    opt2.load_state_dict(saved_opt)
    sch2.load_state_dict(saved_sch)
    run(opt2, sch2, m2, 8, 14)
    assert opt.step_count == opt2.step_count == 14
    for k in FusedLoraAdam8bit._STATE:
        assert torch.equal(getattr(opt, k), getattr(opt2, k)), k
    assert all(torch.equal(p, m2._lora_params[n]) for n, p in m._lora_params.items())


def test_refused_and_ignored_arguments(emu):
    from qflux_b200 import lib
    from qflux_b200.optim import FusedLoraAdam8bit
    m = _model()
    for bad, word in ((dict(amsgrad=True), "amsgrad"), (dict(percentile_clipping=5), "percentile_clipping"),
                      (dict(block_wise=False), "block_wise"), (dict(args=object()), "args")):
        with pytest.raises(lib.QfxError, match=word):
            FusedLoraAdam8bit(m, **bad)
    with pytest.raises(TypeError):
        FusedLoraAdam8bit(m, no_such_argument=1)
    FusedLoraAdam8bit(m, optim_bits=8, is_paged=True)


def test_c_entry_point_refuses_bad_arguments_before_any_cuda_call():
    from qflux_b200 import lib
    L = lib._lib
    p = torch.zeros(4096, dtype=torch.float64)
    vp = lambda t: C.c_void_p(t.data_ptr())
    f = C.c_float

    def call(n_chunks=1, scratch_floats=lib.DET_NORM_PARTIALS, lr=1e-4, step=1, min_8bit=4096, qmap=None):
        return L.qfx_fused_adam8bit(vp(p), vp(p), n_chunks, vp(p), vp(p), 100, vp(p), vp(p), vp(p), vp(p), vp(p), vp(p),
                                    qmap if qmap is not None else vp(p), vp(p), vp(p), vp(p), scratch_floats, f(1.0), f(1.0), f(lr),
                                    f(0.9), f(0.999), f(1e-8), f(0.0), step, min_8bit, None)
    assert call(scratch_floats=lib.DET_NORM_PARTIALS - 1) != 0 and b"scratch" in L.qfx_last_error()
    assert call(lr=-1.0) != 0 and b"lr >= 0" in L.qfx_last_error()
    for kw in (dict(n_chunks=0), dict(step=0), dict(min_8bit=-1), dict(qmap=C.c_void_p(0))):
        assert call(**kw) != 0 and b"bad arguments" in L.qfx_last_error(), kw


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _dp_worker(rank, world, port, out):
    sys.path.insert(0, HERE)
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "qwen-image-finetune_b200"))
    import adam8bit_ref
    from qflux_b200 import lib
    adam8bit_ref.install(lib)
    from qflux_b200.optim import FusedLoraAdam8bit
    from qflux_b200.train_step import _sync_and_step
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    m = _model()
    opt = FusedLoraAdam8bit(m, **CONFIG_ARGS)
    sch = cosine_warmup(opt, warmup=1)
    g = torch.Generator().manual_seed(50 + rank)  # per-rank gradients
    for _ in range(6):
        m.G32.copy_(torch.randn(m.G32.shape, generator=g))
        _sync_and_step(m, opt, 1.0)
        sch.step()
    flat = torch.cat([opt.state1.float(), opt.state2.float(), opt.absmax1, opt.absmax2, opt.s1_32, opt.s2_32] +
                     [p.detach().float().reshape(-1) for p in m.parameters()])
    allp = [torch.zeros_like(flat) for _ in range(world)]
    dist.all_gather(allp, flat)
    if rank == 0:
        torch.save(dict(same=all(torch.equal(allp[0], t) for t in allp), step=opt.step_count), out)
    dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_dp2_ranks_agree_on_codes_absmax_and_parameters(tmp_path):
    out = str(tmp_path / "res.pt")
    mp.spawn(_dp_worker, args=(2, _free_port(), out), nprocs=2, join=True)
    r = torch.load(out)
    assert r["step"] == 6
    assert r["same"], "codes, absmax, fp32 states and every parameter must be identical on both ranks"


def test_gradient_accumulation_2_train_step_equals_restatement_on_the_mean(emu):
    """Two micro-steps of QwenImageEditStep(gradient_accumulation_steps=2) step FusedLoraAdam8bit once on G32 / 2 (the accumulator
    holds the sum): the same parameters, bit for bit, as the restatement fed that mean gradient with the same clip."""
    import adam8bit_ref
    from test_host_orchestration import _inputs, _pair
    from qflux_b200.optim import FusedLoraAdam8bit
    from qflux_b200.train_step import QwenImageEditStep
    x = _inputs(2, 4, 24, 128)
    keys = ("image_latents", "control_latents", "prompt_embeds", "prompt_embeds_mask")
    orc, m = _pair(2, 1, 128, 16, ("to_q", "to_out.0"))
    ps = [torch.nn.Parameter(p.detach().clone()) for p, _ in _members(m)]
    assert max(p.numel() for p in ps) >= 4096
    opt = FusedLoraAdam8bit(m, lr=1e-2)
    ref = adam8bit_ref.Adam8bit(ps, lr=1e-2)
    step = QwenImageEditStep(m, "mse", max_grad_norm=1.0, gradient_accumulation_steps=2)
    for b in range(2):
        emb = {**{k: x[k][b:b + 1] for k in keys}, "img_shapes": x["img_shapes"][b:b + 1]}
        step.train_step(emb, opt, noise=x["noise"][b:b + 1], u=x["u"][b:b + 1])
    assert opt.step_count == 1
    start = [q.detach().clone() for q in ps]
    _restated_step(ref, ps, m, m.G32, 0.5, 1.0)
    for (p, _), q in zip(_members(m), ps):
        assert torch.equal(p.detach(), q.detach())
    assert any(not torch.equal(a, q.detach()) for a, q in zip(start, ps)), "the step must move the parameters"


# ---------------------------------------------------------------------------------------------------- GPU
def _run_case(name):
    r = subprocess.run([sys.executable, CHECK, "--case", name], capture_output=True, text=True, timeout=900, cwd=ROOT)
    res = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
    assert r.returncode == 0 and res, (r.stdout + r.stderr)[-3000:]
    out = json.loads(res[-1][7:])
    assert not out.get("fail"), out
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["kernel_flux_yaml", "kernel_small_and_partial", "repeat_bitwise", "step_qwen", "step_flux_yaml"])
def test_adam8bit_on_gpu(case):
    _run_case(case)
