"""qfx_fused_adamw / qfx_grad_finalize (and their _det variants) per element against tests/adamw_ref.py, the fp64 restatement of
clip_grad_norm_ + torch.optim.AdamW.step, every step from the kernel's own state before it.

    python tools/adamw_check.py [case ...]     (one subprocess per case via tools/harness.py)

  tables_edges      one table of tensors of 1, 4095, 4096, 4097 and 3 x 4096 elements (QFX_ADAMW_CHUNK edges), rank-1 factors and
                    row-strided B views (ld 64) in buffers whose padding columns and guard rows hold a NaN sentinel; guard elements
                    around every tensor's range of the flat gradient / m / v.  Three steps, atomic and det, against the abi mode;
                    sentinels bit-identical.
  hyper_grid        every combination of betas {(0.9, 0.999), (0.9, 0.99), (0.0, 0.999), (0.9, 0.9999)}, eps {1e-8, 1e-3}, weight
                    decay {0, 1e-2, 0.5} (parameters of magnitude 1-4), lr {1e-4, 1e-2}, pre_scale {1, 1/8} and clip {off, norm
                    above max_norm, norm below it}, plus an all-zero gradient: steps 1, 2, 3 from zero moments, then the restated
                    moments at step 999; against the abi and the torch mode.
  grad_finalize     qfx_grad_finalize and _det at n in {1, 255, 257, 2^20 + 3, the flat size of each bench config}: out equals
                    bf16(g pre_scale coef) with coef from the kernel's own sumsq (bit for bit without a clip; one-ulp flips only
                    next to rounding midpoints with one), sumsq within RED_TOL of sum |terms| of fp64, guards untouched, and det /
                    atomic outputs identical whenever their sumsq bits agree.
  bench_size_qwen_edit / bench_size_flux_kontext
                    the flat gradient and tables of bench.py's adapters (Qwen-Image-Edit r = 16 on to_q / to_k / to_v / to_out.0 of
                    60 blocks; FLUX-Kontext r = 32 with the YAML targets, 172 M elements), three steps, atomic and det from the same
                    state: both against the abi mode, and bit-identical to each other whenever their sumsq bits agree (always
                    on the third step, which does not clip).
  optimizer_contract
                    FusedLoraAdamW on a tiny Qwen model over 20 steps of the cosine warm-up schedule (first lr 0: moments and step
                    advance, parameters do not move), grad_divisor = 4, a state_dict round trip at step 7, the deterministic flag
                    on and off, finalize_grads' bf16 `param.grad`s; and the trajectory against fp64 no further than 1.5 x that
                    of clip_grad_norm_ + torch.optim.AdamW on bf16 parameters (what the reference trainer runs) + 1e-2.
Each case returns its measurements plus `fail`, the list of violated checks.
"""
import itertools
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "qwen-image-finetune_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import harness  # noqa: E402

BETAS = ((0.9, 0.999), (0.9, 0.99), (0.0, 0.999), (0.9, 0.9999))
EPSS = (1e-8, 1e-3)
WDS = (0.0, 1e-2, 0.5)
LRS = (1e-4, 1e-2)
PRE_SCALES = (1.0, 0.125)
CLIPS = (("off", 0.0, 4.0), ("above", 1.0, 4.0), ("below", 1.0, 0.5))  # (name, max_norm, norm of grad * pre_scale)
STEPS = (1, 2, 3, 999)
CHECK_CHUNK = 1 << 24


def grid():
    """(name, hp, target norm, zero gradient) of every hyper_grid point"""
    pts = []
    for (b1, b2), eps, wd, lr, ps, (cn, mx, norm) in itertools.product(BETAS, EPSS, WDS, LRS, PRE_SCALES, CLIPS):
        hp = dict(lr=lr, beta1=b1, beta2=b2, eps=eps, weight_decay=wd, pre_scale=ps, max_norm=mx)
        pts.append((f"b{b1}_{b2}_eps{eps}_wd{wd}_lr{lr}_ps{ps}_clip{cn}", hp, norm, False))
    pts.append(("zero_grad", dict(lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=1e-2, pre_scale=1.0, max_norm=1.0), 0.0, True))
    return pts


def grid_problem(n, seed, device):
    """parameters of magnitude 1-4 (random sign, so the decay is visible), gradient directions with log-uniform magnitudes over four
    decades and a positive mean (so a slip in the step's size moves the signed mean error), unit norm"""
    import torch
    g = torch.Generator(device="cpu").manual_seed(seed)
    sgn = lambda: torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0)
    p = (sgn() * (1 + 3 * torch.rand(n, generator=g))).to(torch.bfloat16)
    d = torch.where(torch.rand(n, generator=g) < 0.7, 1.0, -1.0) * 10 ** (-4 * torch.rand(n, generator=g))
    return p.to(device), (d / d.norm()).float().to(device)


def run_grid(step_fn, n, device, modes=("abi", "torch"), stop_at_first_failure=False, points=None):
    """step_fn(p, g, m, v, hp, step) -> sumsq (float): one fused step in place on flat p (bf16), m, v (fp32).  Every grid point runs
    steps 1, 2, 3 from zero moments, then step 999 from the fp64-restated moments after step 3.  Returns (stats, failures)."""
    import torch
    import adamw_ref as ar
    stats, fail = dict(points=0, m_max_ulps=0.0, v_max_ulps=0.0, flip_frac_max=0.0, flips=0, elements=0, mean_err_ulps_max=0.0,
                       torch_sqrt_bc2_rel_gap_b2_9999=0.0, torch_flip_frac_max=0.0), []
    for k, (name, hp, norm, zero) in enumerate(points or grid()):
        p0, d = grid_problem(n, 100 + k, device)
        p, m, v = p0.clone(), torch.zeros(n, device=device), torch.zeros(n, device=device)
        g = torch.zeros(n, device=device) if zero else (d * (norm / hp["pre_scale"])).float()
        stats["points"] += 1
        for step in STEPS:
            if step == 999:  # the restated moments after step 3, rounded to fp32
                S = ar.scalars("abi", hp["lr"], hp["beta1"], hp["beta2"], hp["eps"], hp["weight_decay"], 3, hp["pre_scale"],
                               hp["max_norm"])
                R = ar.step_ref(before["p"], before["g"], before["m"], before["v"], S, sumsq=ss)
                m.copy_(R["m"].float())
                v.copy_(R["v"].float())
            before = dict(p=p.clone(), g=g.clone(), m=m.clone(), v=v.clone())
            ss = step_fn(p, g, m, v, hp, step)
            after = dict(p=p, m=m, v=v)
            for mode in modes:
                st, f = ar.check_step(before, after, hp, step, ss, mode, tag=f"{name}: ")
                fail += f
                if mode == "abi":
                    stats["m_max_ulps"] = max(stats["m_max_ulps"], st["m_max_ulps"])
                    stats["v_max_ulps"] = max(stats["v_max_ulps"], st["v_max_ulps"])
                    stats["flip_frac_max"] = max(stats["flip_frac_max"], st["flip_frac"])
                    stats["flips"] += st["flips"]
                    stats["elements"] += st["n"]
                    stats["mean_err_ulps_max"] = max(stats["mean_err_ulps_max"], abs(st["mean_err_ulps"] - st["ideal_mean_err_ulps"]))
                else:
                    stats["torch_flip_frac_max"] = max(stats["torch_flip_frac_max"], st["flip_frac"])
            if hp["beta2"] == 0.9999:
                a = ar.scalars("abi", 1, 0, hp["beta2"], 0, 0, step)["bc2_sqrt"]
                t = ar.scalars("torch", 1, 0, hp["beta2"], 0, 0, step)["bc2_sqrt"]
                stats["torch_sqrt_bc2_rel_gap_b2_9999"] = max(stats["torch_sqrt_bc2_rel_gap_b2_9999"], abs(a - t) / t)
            if fail and stop_at_first_failure:
                stats["first_failure"] = name
                return stats, fail
    return stats, fail


# ---------------------------------------------------------------------------------------------------- GPU helpers
def _flat_p(params):
    import torch
    return torch.cat([q.reshape(-1) for q in params])


def _checks(before, after, hp, step, ss, res, fail, tag, modes=("abi",)):
    """adamw_ref.check_step over CHECK_CHUNK slices of the flat state; folds the statistics into res[tag]"""
    import adamw_ref as ar
    n = before["p"].numel()
    agg = res.setdefault(tag, dict(m_max_ulps=0.0, v_max_ulps=0.0, flips=0, elements=0))
    sums = res.setdefault("_sums_" + tag, [0.0, 0.0])
    for mode in modes:
        for lo in range(0, n, CHECK_CHUNK):
            sl = slice(lo, min(n, lo + CHECK_CHUNK))
            st, f = ar.check_step({k: t[sl] for k, t in before.items()}, {k: t[sl] for k, t in after.items()}, hp, step, ss, mode,
                                  tag=f"{tag}: ")
            fail += f
            if mode != "abi":
                continue
            agg["m_max_ulps"] = max(agg["m_max_ulps"], st["m_max_ulps"])
            agg["v_max_ulps"] = max(agg["v_max_ulps"], st["v_max_ulps"])
            agg["flips"] += st["flips"]
            sums[0] += st["mean_err_ulps"] * st["n"]
            sums[1] += st["ideal_mean_err_ulps"] * st["n"]
            agg["elements"] += st["n"]
    agg["flip_frac"] = agg["flips"] / max(agg["elements"], 1)
    agg["signed_mean_err_ulps"] = sums[0] / max(agg["elements"], 1)
    agg["ideal_signed_mean_err_ulps"] = sums[1] / max(agg["elements"], 1)


def _bits(t):
    import torch
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _same_bits(a, b):
    import torch
    return torch.equal(_bits(a), _bits(b))


def hyper_grid():
    import torch
    from qflux_b200 import lib
    n = 256 * 64
    buf = torch.zeros(256, 64, device="cuda", dtype=torch.bfloat16)
    tables = lib.adamw_tables([(buf, 0)], "cuda")
    sumsq = torch.zeros(1, device="cuda")

    def step_fn(p, g, m, v, hp, step):
        buf.view(-1).copy_(p)
        lib.fused_adamw(tables, g, m, v, sumsq, hp["pre_scale"], hp["max_norm"], hp["lr"], hp["beta1"], hp["beta2"], hp["eps"],
                        hp["weight_decay"], step)
        p.copy_(buf.view(-1))
        return float(sumsq)
    stats, fail = run_grid(step_fn, n, "cuda")
    stats["fail"] = fail[:20]
    stats["failures"] = len(fail)
    return stats


def tables_edges():
    import torch
    from gemm_tile_check import SENT_F32, is_sent, sentinel
    from qflux_b200 import lib
    gen = torch.Generator(device="cuda").manual_seed(5)
    # (rows, cols, B view of a 64-column buffer?): sizes 1, 4095, 4096, 4097, 3 x 4096, rank-1 A and B, row-strided B views
    shapes = [(1, 1, True), (45, 91, False), (16, 256, False), (241, 17, True), (768, 16, True), (1, 300, False), (300, 1, True),
              (257, 16, True)]
    GUARD, GROWS = 5, 2
    params, bufs, members, off = [], [], [], GUARD
    for rows, cols, strided in shapes:
        vals = ((1 + 3 * torch.rand(rows, cols, device="cuda", generator=gen)) *
                torch.where(torch.rand(rows, cols, device="cuda", generator=gen) < 0.5, -1.0, 1.0)).bfloat16()
        if strided:
            b = sentinel(rows + GROWS, 64, device="cuda")
            b[:rows, :cols] = vals
            p = b[:rows, :cols]
            bufs.append((b, rows, cols))
        else:
            p = vals
        params.append(p)
        members.append((p, off))
        off += p.numel() + GUARD
    n = off
    tables = lib.adamw_tables(members, "cuda")
    used = torch.zeros(n, dtype=torch.bool, device="cuda")
    for p, o in members:
        used[o: o + p.numel()] = True
    G = torch.where(used, torch.randn(n, device="cuda", generator=gen) * 0.05, torch.full((n,), 0.5, device="cuda"))
    hp = dict(lr=1e-2, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=1e-2, pre_scale=0.5, max_norm=1.0)
    res, fail = dict(elements=int(used.sum()), tensors=len(members), chunks=int(tables[1].shape[0])), []
    ss = torch.zeros(1, device="cuda")
    scratch = torch.zeros(lib.DET_NORM_PARTIALS, device="cuda")
    for variant in ("atomic", "det"):
        m = torch.full((n,), SENT_F32, device="cuda").masked_fill(used, 0.0)
        v = torch.full((n,), SENT_F32, device="cuda").masked_fill(used, 0.0)
        start = [p.clone() for p in params]
        for step in (1, 2, 3):
            before = dict(p=_flat_p(params), g=torch.cat([G[o: o + p.numel()] for p, o in members]),
                          m=torch.cat([m[o: o + p.numel()] for p, o in members]), v=torch.cat([v[o: o + p.numel()] for p, o in members]))
            args = (tables, G, m, v, ss, hp["pre_scale"], hp["max_norm"], hp["lr"], hp["beta1"], hp["beta2"], hp["eps"],
                    hp["weight_decay"], step)
            lib.fused_adamw(*args) if variant == "atomic" else lib.fused_adamw_det(*args, scratch=scratch)
            want_ss = float((G.double() * hp["pre_scale"]).pow(2).sum())
            if abs(float(ss) - want_ss) > 1e-5 * want_ss:
                fail.append(f"{variant} step {step}: sumsq {float(ss)} vs fp64 {want_ss} (guards included)")
            after = dict(p=_flat_p(params), m=torch.cat([m[o: o + p.numel()] for p, o in members]),
                         v=torch.cat([v[o: o + p.numel()] for p, o in members]))
            _checks(before, after, hp, step, float(ss), res, fail, variant)
        if not (bool((m[~used] == SENT_F32).all()) and bool((v[~used] == SENT_F32).all())):
            fail.append(f"{variant}: m / v guard elements written")
        for b, rows, cols in bufs:
            if not (bool(is_sent(b[:, cols:]).all()) and bool(is_sent(b[rows:]).all())):
                fail.append(f"{variant}: padding columns / guard rows of a {rows} x {cols} B view written")
        if not any(not torch.equal(a, p) for a, p in zip(start, params)):
            fail.append(f"{variant}: no parameter moved")
        res.pop("_sums_" + variant)
        with torch.no_grad():  # the det variant starts from the same parameters
            for p, s0 in zip(params, start):
                p.copy_(s0)
    res["fail"] = fail
    return res


def _gfin_one(n, pre_scale, max_norm, res, fail, seed):
    import torch
    from glue_check import RED_TOL
    import adamw_ref as ar
    from qflux_b200 import lib
    GU = 8
    gen = torch.Generator(device="cuda").manual_seed(seed)
    g = torch.randn(n, device="cuda", generator=gen) * (4.0 / max(n, 1) ** 0.5)
    SENT = torch.tensor(-7.25).bfloat16().item()
    outs = {}
    sss = {}
    scratch = torch.zeros(lib.DET_NORM_PARTIALS, device="cuda")
    for variant in ("atomic", "det"):
        full = torch.full((n + 2 * GU,), SENT, device="cuda", dtype=torch.bfloat16)
        out = full[GU: GU + n]
        ss = torch.zeros(1, device="cuda")
        if variant == "atomic":
            lib.grad_finalize(g, pre_scale, max_norm, ss, out)
        else:
            lib.grad_finalize_det(g, pre_scale, max_norm, ss, out, scratch=scratch)
        torch.cuda.synchronize()
        tag = f"{variant}_n{n}_ps{pre_scale}_mx{max_norm}"
        if not (bool((full[:GU] == SENT).all()) and bool((full[GU + n:] == SENT).all())):
            fail.append(f"{tag}: guard elements written")
        x = g.double() * pre_scale
        want = float((x * x).sum())
        if abs(float(ss) - want) > RED_TOL * want:
            fail.append(f"{tag}: sumsq {float(ss)!r} vs fp64 {want!r}")
        coef = ar.clip_coef(float(ss), float(ar._f32(max_norm)))
        exact = x * coef
        r = exact.to(torch.bfloat16)
        flip = out != r
        if coef == 1.0:  # no clip: g * pre_scale is exact in fp32 (pre_scale a power of two), its bf16 rounding bit for bit
            bad = int(flip.sum())
        else:  # fast-math sqrtf / division in the coefficient: flips allowed within 2^-20 |x| of a midpoint, to the other side
            nb = ar.bf16_neighbour(r, exact)
            near = ((exact - (r.double() + nb.double()) / 2).abs() <= 2.0 ** -20 * exact.abs()) & (nb != r)
            bad = int((flip & ~(near & (out == nb))).sum())
        ps = dict(flips=int(flip.sum()), bad=bad)
        res[tag] = dict(sumsq_rel_err=abs(float(ss) - want) / max(want, 1e-300), flips=ps["flips"], flip_frac=ps["flips"] / n,
                        clipped=coef < 1.0)
        if ps["bad"]:
            fail.append(f"{tag}: {ps['bad']} elements differ from bf16(g pre_scale coef) away from a rounding midpoint")
        outs[variant], sss[variant] = out.clone(), ss.clone()
    same_ss = _same_bits(sss["atomic"], sss["det"])
    res[f"n{n}_ps{pre_scale}_mx{max_norm}_sumsq_bits_agree"] = same_ss
    if (same_ss or max_norm <= 0) and not _same_bits(outs["atomic"], outs["det"]):
        fail.append(f"n{n}: det and atomic outputs differ with the same sumsq")


def grad_finalize():
    import prodigy_check as pc
    res, fail = {}, []
    sizes = [1, 255, 257, (1 << 20) + 3, 60 * 4 * 2 * 3072 * 16, sum(32 * (a + b) for a, b in pc._flux_yaml_shapes())]
    for i, n in enumerate(sizes):
        for ps, mx in ((1.0, 0.0), (0.5, 1.0), (0.125, 1e3)):
            _gfin_one(n, ps, mx, res, fail, 10 + i)
    res["fail"] = fail
    return res


def _bench_size(shapes, r, hp_steps):
    import torch
    import prodigy_check as pc
    from qflux_b200 import lib
    fl = pc.FlatLora(shapes, r, 11)
    n = fl.n
    tables = lib.adamw_tables(fl.members, "cuda")
    m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    ss_a, ss_d = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    scratch = torch.zeros(lib.DET_NORM_PARTIALS, device="cuda")
    res, fail = dict(elements=n, tensors=len(fl.members)), []
    for step, hp in enumerate(hp_steps, 1):
        G = fl.grads(step, 5)
        p0, m0, v0 = [p.clone() for p in fl.params], m.clone(), v.clone()
        before = dict(p=_flat_p(fl.params), g=G, m=m0, v=v0)
        args = lambda ss: (tables, G, m, v, ss, hp["pre_scale"], hp["max_norm"], hp["lr"], hp["beta1"], hp["beta2"], hp["eps"],
                           hp["weight_decay"], step)
        lib.fused_adamw_det(*args(ss_d), scratch=scratch)
        det = dict(p=_flat_p(fl.params), m=m.clone(), v=v.clone())
        _checks(before, det, hp, step, float(ss_d), res, fail, "det")
        with torch.no_grad():  # the atomic variant from the same state
            for p, s0 in zip(fl.params, p0):
                p.copy_(s0)
        m.copy_(m0)
        v.copy_(v0)
        lib.fused_adamw(*args(ss_a))
        ato = dict(p=_flat_p(fl.params), m=m, v=v)
        _checks(before, ato, hp, step, float(ss_a), res, fail, "atomic")
        want = float((G.double() * hp["pre_scale"]).pow(2).sum())
        res[f"step{step}_sumsq_rel_err"] = [abs(float(s) - want) / want for s in (ss_a, ss_d)]
        same_ss = _same_bits(ss_a, ss_d)
        res[f"step{step}_sumsq_bits_agree"] = same_ss
        if same_ss or hp["max_norm"] <= 0:
            if not all(_same_bits(det[k], ato[k]) for k in ("p", "m", "v")):
                fail.append(f"step {step}: det and atomic states differ with the same clip")
        if step == len(hp_steps) and hp["max_norm"] > 0:
            fail.append("the last step must not clip (it compares det and atomic unconditionally)")
    if any(bool(b[:, fl.r:].any()) for b in fl.bufs):
        fail.append("B padding columns written")
    res = {k: v for k, v in res.items() if not k.startswith("_sums_")}
    res["fail"] = fail
    return res


BENCH_HP = dict(lr=1e-4, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=1e-2, pre_scale=0.5, max_norm=1.0)
BENCH_STEPS = (BENCH_HP, BENCH_HP, dict(BENCH_HP, max_norm=0.0))


def bench_size_qwen_edit():
    return _bench_size([(3072, 3072)] * 4 * 60, 16, BENCH_STEPS)


def bench_size_flux_kontext():
    import prodigy_check as pc
    return _bench_size(pc._flux_yaml_shapes(), 32, BENCH_STEPS)


# ---------------------------------------------------------------------------------------------------- FusedLoraAdamW
def _tiny_qwen(seed=7):
    import torch
    from qflux_b200.qwen_model import QwenB200Config, QwenImageB200
    torch.manual_seed(seed)
    m = QwenImageB200(QwenB200Config(num_layers=1, num_attention_heads=2, joint_attention_dim=128))
    m.add_adapter(4, 4, b_std=0.05)
    return m


class Problem:
    """grad(p) = 4 a (p - target) + noise_t per LoRA tensor (fp64): a loss each run descends from its own parameters, fixed draws"""

    def __init__(self, params, seed=3):
        import torch
        g = torch.Generator().manual_seed(seed)
        self.target = {n: p.detach().double().cpu() + torch.randn(p.shape, generator=g, dtype=torch.float64) for n, p in params.items()}
        self.a = {n: torch.rand(p.shape, generator=g, dtype=torch.float64) + 0.5 for n, p in params.items()}
        self.seed = seed

    def grads(self, params, t):
        import torch
        g = torch.Generator().manual_seed(self.seed * 1000 + t)
        return {n: (self.a[n] * (p.detach().double().cpu() - self.target[n]) * 4 +
                    0.1 * torch.randn(p.shape, generator=g, dtype=torch.float64)).to(p.device)
                for n, p in params.items()}


HP = dict(lr=2e-2, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)
MAX_NORM, STEPS_N, WARMUP = 1.0, 20, 5


def _fused_run(m, prob, det, t0=0, t1=STEPS_N, opt=None, sch=None, scale=1.0, stop_at=None):
    import torch
    import adamw_ref as ar
    from qflux_b200.optim import FusedLoraAdamW
    opt = opt or FusedLoraAdamW(m, **HP, max_grad_norm=MAX_NORM)
    sch = sch or ar.cosine_warmup(opt, WARMUP, STEPS_N)
    views = m.lora_grad_views()
    torch.use_deterministic_algorithms(det)
    try:
        for t in range(t0, t1):
            for n, g in prob.grads(m._lora_params, t).items():
                views[n].copy_(g * scale)
            opt.step(grad_divisor=scale if scale != 1.0 else None)
            sch.step()
    finally:
        torch.use_deterministic_algorithms(False)
    return opt, sch


def _restated_run(start, prob, dtype):
    import torch
    import adamw_ref as ar
    ps = {n: torch.nn.Parameter(p.detach().to(dtype).clone()) for n, p in start.items()}
    opt = torch.optim.AdamW(list(ps.values()), **HP)
    sch = ar.cosine_warmup(opt, WARMUP, STEPS_N)
    for t in range(STEPS_N):
        for n, g in prob.grads(ps, t).items():
            ps[n].grad = g.to(dtype)
        torch.nn.utils.clip_grad_norm_(list(ps.values()), MAX_NORM)  # BaseTrainer.clip_gradients
        opt.step()
        sch.step()
    return ps


def optimizer_contract():
    import copy
    import torch
    from qflux_b200.optim import FusedLoraAdamW
    res, fail = {}, []
    # the first warm-up step has lr 0: the moments and the step count advance, the parameters do not move
    m = _tiny_qwen()
    start = {n: p.detach().clone() for n, p in m._lora_params.items()}
    prob = Problem(m._lora_params)
    opt, sch = _fused_run(m, prob, True, 0, 1)
    if not (opt.step_count == 1 and bool(opt.exp_avg.any()) and bool(opt.exp_avg_sq.any())):
        fail.append("lr = 0 step: moments / step count did not advance")
    if not all(torch.equal(p, start[n]) for n, p in m._lora_params.items()):
        fail.append("lr = 0 step moved a parameter")
    _fused_run(m, prob, True, 1, 7, opt, sch)
    saved = copy.deepcopy(opt.state_dict()), copy.deepcopy(sch.state_dict()), {n: p.detach().clone() for n, p in m._lora_params.items()}
    _fused_run(m, prob, True, 7, STEPS_N, opt, sch)
    final_det = {n: p.detach().clone() for n, p in m._lora_params.items()}
    # state_dict round trip at step 7 continues bit for bit (deterministic flag on: the clip's norm is summed in a fixed order)
    m2 = _tiny_qwen()
    with torch.no_grad():
        for n, p in m2._lora_params.items():
            p.copy_(saved[2][n])
    opt2 = FusedLoraAdamW(m2, **HP, max_grad_norm=MAX_NORM)
    import adamw_ref as ar
    sch2 = ar.cosine_warmup(opt2, WARMUP, STEPS_N)
    opt2.load_state_dict(saved[0])
    sch2.load_state_dict(saved[1])
    _fused_run(m2, prob, True, 7, STEPS_N, opt2, sch2)
    res["resume_bit_exact"] = all(torch.equal(p, final_det[n]) for n, p in m2._lora_params.items()) and \
        torch.equal(opt.exp_avg, opt2.exp_avg) and torch.equal(opt.exp_avg_sq, opt2.exp_avg_sq) and opt2.step_count == STEPS_N
    if not res["resume_bit_exact"]:
        fail.append("state_dict round trip at step 7 does not continue bit for bit")
    # grad_divisor = 4 on four times the gradient: the same bits (flag on)
    m3 = _tiny_qwen()
    _fused_run(m3, prob, True, scale=4.0)
    res["grad_divisor_4_bit_exact"] = all(torch.equal(p, final_det[n]) for n, p in m3._lora_params.items())
    if not res["grad_divisor_4_bit_exact"]:
        fail.append("grad_divisor = 4 on 4 x the gradient differs from the plain run")
    # flag off: the same accuracy
    m4 = _tiny_qwen()
    _fused_run(m4, prob, False)
    final_atomic = {n: p.detach().clone() for n, p in m4._lora_params.items()}
    # against fp64 and against clip_grad_norm_ + torch.optim.AdamW on bf16 parameters
    p64 = _restated_run(start, prob, torch.float64)
    p16 = _restated_run(start, prob, torch.bfloat16)
    for tag, final in (("det", final_det), ("atomic", final_atomic)):
        worst, bad = 0.0, []
        for n, s0 in start.items():
            disp = (p64[n].detach() - s0.double()).norm()
            e_f = float((final[n].double() - p64[n].detach()).norm() / disp)
            e_b = float((p16[n].detach().double() - p64[n].detach()).norm() / disp)
            worst = max(worst, e_f)
            if not e_f <= 1.5 * e_b + 1e-2:
                bad.append(f"{tag} {n}: {e_f:.3e} vs bf16 torch.optim.AdamW {e_b:.3e}")
        res[f"{tag}_worst_err_vs_fp64"] = worst
        fail += bad[:5]
    # finalize_grads: every param.grad is the bf16 of its own slice of G32 (one rank, no clip)
    views = m.lora_grad_views()
    for n, g in prob.grads(m._lora_params, 99).items():
        views[n].copy_(g)
    m.finalize_grads(1, 0.0)
    torch.cuda.synchronize()
    res["finalize_exact"] = all(torch.equal(p.grad, views[n].to(torch.bfloat16)) for n, p in m._lora_params.items())
    if not res["finalize_exact"]:
        fail.append("finalize_grads: a param.grad is not the bf16 of its G32 slice")
    res["fail"] = fail
    return res


CASES = dict(tables_edges=tables_edges, hyper_grid=hyper_grid, grad_finalize=grad_finalize, bench_size_qwen_edit=bench_size_qwen_edit,
             bench_size_flux_kontext=bench_size_flux_kontext, optimizer_contract=optimizer_contract)

if __name__ == "__main__":
    harness.main(CASES, os.path.abspath(__file__), "adamw_check.log")
