"""qfx_fused_adam8bit / FusedLoraAdam8bit on the GPU against tests/adam8bit_ref.py, the plain-torch restatement of bitsandbytes'
block-wise `Adam8bit`.

    python tools/adam8bit_check.py [case ...]     (one subprocess per case via tools/harness.py)

  kernel_flux_yaml  the kernel on random flat buffers laid out like the FLUX-Kontext YAML target set at r = 32 (990 tensors, 172 M
                    elements, every B factor a row-strided view of a 64-column buffer, the 64-wide embedder's A on the fp32 path), the
                    configs' init_args, 20 steps of a cosine warm-up from lr 0 with the clip active.  Every step is checked against the
                    restatement started from the kernel's own state before it (and the kernel's own ||g||^2):
                      - absmax within 1e-6 relative; fp32 states within 2^-21 of their terms' magnitude;
                      - codes equal, except that a code may lie anywhere between the codes of the restated state pushed down and up by
                        its rounding allowance (2^-21 of |beta s| + |(1 - beta) g|, plus 2^-21 of s / absmax): the kernel runs with
                        --use_fast_math and contracts to FMA, so a state within a few fp32 ulps of a decision boundary (the midpoint
                        between two codes, or 0 for state1's sign rule) may land on either side.  The share of codes that differ at
                        all is reported and must stay below 1e-4;
                      - bf16 parameters equal, or within the roundings of the restated fp32 result moved by 2^-20 of the update plus
                        two fp32 ulps of the parameter; the share that differs is reported.
                    After the 20 steps the parameters' rel-L2 against a free-running restatement must be <= 1e-3.
  kernel_small_and_partial
                    the same checks on the boundary shapes: numel 4095 (fp32 path) and 4096 (8-bit), 5000 elements (partial last
                    block), a row-strided [300, 16] view of a [300, 64] buffer whose padding must stay zero, and a block of the
                    4096-element tensor whose gradient is always zero (absmax 0, zero codes; its parameters only decay), with
                    weight_decay 0.01.  The CPU suite
                    runs this case on the emulation (`kernel_small_and_partial("cpu")`).
  repeat_bitwise    the FLUX-YAML steps twice from the same state: parameters, codes, absmax and fp32 states agree bit for bit.
  step_qwen / step_flux_yaml
                    three `train_step`s with FusedLoraAdam8bit (2-block full-width Qwen-Image-Edit, every site; FLUX 2 double + 2 single
                    blocks, YAML targets): loss and parameters finite, and the parameters within 1e-2 (rel-L2 of the difference over the
                    displacement) of the restatement fed the gradient each step left in G32, with at most 1e-3 of the codes differing.
"""
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "qwen-image-finetune_b200"), os.path.join(ROOT, "tools"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import harness  # noqa: E402

ARGS = dict(lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0)  # the configs' init_args, bitsandbytes' defaults for the rest
MIN_8BIT = 4096
TOL = 2.0 ** -21


def cosine_lrs(lr, steps=20, warmup=5):
    """diffusers' get_cosine_schedule_with_warmup (the configs' `scheduler_type: cosine`): starts at lr 0"""
    return [lr * (t / warmup if t < warmup else 0.5 * (1 + math.cos(math.pi * (t - warmup) / (steps - warmup)))) for t in range(steps)]


class Flat:
    """FusedLoraAdam8bit's buffers for `members` ((bf16 param, grad offset) pairs), plus per-element maps for the restatement."""

    def __init__(self, members, n, dev):
        import torch
        import adam8bit_ref
        from qflux_b200 import lib
        self.members, self.n, self.dev = members, n, dev
        offsets, na, ns = lib.adam8bit_layout(members, MIN_8BIT)
        self.offsets = torch.tensor(offsets, dtype=torch.int64).to(dev)
        self.tables = lib.adamw_tables(members, dev)
        z = lambda k, dt=torch.float32: torch.zeros(max(1, k), device=dev, dtype=dt)
        self.st = dict(state1=z(n, torch.uint8), state2=z(n, torch.uint8), absmax1=z(na), absmax2=z(na), s1_32=z(ns), s2_32=z(ns))
        self.q1, self.q2 = adam8bit_ref.create_dynamic_map(True).to(dev), adam8bit_ref.create_dynamic_map(False).to(dev)
        self.bw = torch.zeros(n, dtype=torch.bool, device=dev)     # element of an 8-bit tensor
        self.idx = torch.zeros(n, dtype=torch.int64, device=dev)   # its absmax block, or its fp32 state element
        for (p, off), so in zip(members, offsets):
            k = p.numel()
            r = torch.arange(k, device=dev)
            self.bw[off: off + k] = k >= MIN_8BIT
            self.idx[off: off + k] = so + (r // adam8bit_ref.BLOCK if k >= MIN_8BIT else r)
        self.sumsq = torch.zeros(1, device=dev)
        self.scratch = torch.zeros(lib.DET_NORM_PARTIALS, device=dev)

    def params(self):
        import torch
        out = torch.zeros(self.n, device=self.dev, dtype=torch.bfloat16)
        for p, off in self.members:
            out[off: off + p.numel()] = p.reshape(-1)
        return out

    def step(self, G, lr, t, args=ARGS, max_norm=1.0):
        from qflux_b200 import lib
        s = self.st
        lib.fused_adam8bit(self.tables, self.offsets, G, s["state1"], s["state2"], s["absmax1"], s["absmax2"], s["s1_32"], s["s2_32"],
                           self.q1, self.q2, self.sumsq, self.scratch, 1.0, max_norm, lr, args["betas"][0], args["betas"][1], args["eps"],
                           args["weight_decay"], t, MIN_8BIT)


def restate(fl, st, p, G, sumsq, lr, t, args=ARGS, max_norm=1.0):
    """One restated step on flat buffers from state `st` and bf16 parameters `p` (flat, grad layout), with the clip coefficient formed
    in fp32 from `sumsq`.  Returns (new state, new parameters, rounding allowances: terms1, terms2 of the states, the update)."""
    import numpy as np
    import torch
    import adam8bit_ref as ar
    f = np.float32
    coef = min(f(max_norm) / (f(np.sqrt(f(sumsq))) + f(1e-6)), f(1)) if max_norm > 0 else f(1)
    g = G * torch.tensor(coef, dtype=torch.float32)
    sc = ar.scalars(lr, args["betas"][0], args["betas"][1], args["eps"], args["weight_decay"], t)
    bw, sm, idx = fl.bw, ~fl.bw, fl.idx
    o1, o2 = torch.empty_like(g), torch.empty_like(g)
    o1[bw] = fl.q1[st["state1"][bw].long()] * st["absmax1"][idx[bw]]
    o2[bw] = fl.q2[st["state2"][bw].long()] * st["absmax2"][idx[bw]]
    o1[sm], o2[sm] = st["s1_32"][idx[sm]], st["s2_32"][idx[sm]]
    w, s1, s2 = torch.empty_like(p), torch.empty_like(g), torch.empty_like(g)
    for mask, blockwise in ((bw, True), (sm, False)):
        w[mask], s1[mask], s2[mask] = ar.update(p[mask], g[mask], o1[mask], o2[mask], sc, blockwise)
    new = {k: v.clone() for k, v in st.items()}
    a1 = torch.zeros_like(st["absmax1"]).scatter_reduce_(0, idx[bw], s1[bw].abs(), "amax")
    a2 = torch.zeros_like(st["absmax2"]).scatter_reduce_(0, idx[bw], s2[bw].abs(), "amax")
    new["absmax1"], new["absmax2"] = a1, a2
    e1, e2 = a1[idx[bw]], a2[idx[bw]]
    new["state1"][bw] = torch.where(e1 > 0, code1(fl.q1, s1[bw] / e1), ar.CODE1_ZERO).to(torch.uint8)
    new["state2"][bw] = torch.where(e2 > 0, ar.quantize(fl.q2, s2[bw] / e2), ar.CODE2_ZERO).to(torch.uint8)
    new["s1_32"][idx[sm]], new["s2_32"][idx[sm]] = s1[sm], s2[sm]
    b1, b2 = sc["beta1"], sc["beta2"]
    terms1 = (o1 * b1).abs() + ((1 - b1) * g).abs()
    terms2 = (o2 * b2).abs() + (1 - b2) * g * g
    upd = sc["step_size"] * (s1 / (s2.sqrt() + sc["c2eps"]))
    return new, w, dict(s1=s1, s2=s2, terms1=terms1, terms2=terms2, w32=p.float() + upd, upd=upd, decay=sc["decay"])


def code1(q1, x):
    """state1's code for x = s1 / absmax: the nearest entry, then bitsandbytes' sign rule (monotone in x)"""
    import torch
    import adam8bit_ref as ar
    c = ar.quantize(q1, x)
    return c + torch.where(torch.signbit(q1[c]) != torch.signbit(x), torch.where(x > 0, 1, -1), 0)


def compare_step(fl, got, got_p, want, want_p, aux, acc):
    """The kernel's state and parameters after one step against the restatement from the same state (the bands of the docstring)."""
    import torch
    import adam8bit_ref as ar
    bw, sm, idx = fl.bw, ~fl.bw, fl.idx
    fail = acc["fail"]
    for k in ("absmax1", "absmax2"):
        err = float(((got[k] - want[k]).abs() / want[k].clamp_min(1e-30)).max())
        acc["absmax_err"] = max(acc["absmax_err"], err)
        if not err <= 1e-6:
            fail.append(f"{k}: {err:.3e} relative")
    for k, s, terms in (("s1_32", "s1", "terms1"), ("s2_32", "s2", "terms2")):
        d = (got[k][idx[sm]] - aux[s][sm]).abs()
        if bool((d > TOL * aux[terms][sm] + 1e-38).any()):
            fail.append(f"{k} outside 2^-21 of its terms")
    for k, s, terms, a, fn in (("state1", "s1", "terms1", want["absmax1"], lambda x: code1(fl.q1, x)),
                               ("state2", "s2", "terms2", want["absmax2"], lambda x: ar.quantize(fl.q2, x))):
        sv, eps, e = aux[s][bw], TOL * aux[terms][bw], a[idx[bw]]
        x = sv / e
        lo, hi = fn((sv - eps) / e - TOL * x.abs()), fn((sv + eps) / e + TOL * x.abs())
        zero = ar.CODE1_ZERO if k == "state1" else ar.CODE2_ZERO
        lo, hi = torch.where(e > 0, lo, zero), torch.where(e > 0, hi, zero)
        c = got[k][bw].long()
        diff = int((c != want[k][bw].long()).sum())
        out = int(((c < lo) | (c > hi)).sum())
        acc[k + "_differ"] += diff
        if out:
            fail.append(f"{k}: {out} codes outside the rounding band")
    w32, upd = aux["w32"], aux["upd"]
    ulp = torch.finfo(torch.float32).eps * w32.abs()
    d = TOL * 2 * upd.abs() + 2 * ulp
    dec = lambda v: (v.to(torch.bfloat16).float() * aux["decay"]).to(torch.bfloat16).float()
    lo, hi = dec(w32 - d), dec(w32 + d)
    gp = got_p.float()
    acc["params_differ"] += int((got_p != want_p).sum())
    out = int(((gp < torch.minimum(lo, hi)) | (gp > torch.maximum(lo, hi))).sum())
    if out:
        fail.append(f"{out} parameters outside their rounding band")
    acc["elements"] += fl.n


def check_run(fl, grads, lrs, args=ARGS, free_tol=1e-3):
    """The kernel over the steps, each checked against the restatement from the kernel's own state, then against a free run."""
    import torch
    acc = dict(fail=[], absmax_err=0.0, state1_differ=0, state2_differ=0, params_differ=0, elements=0)
    start = fl.params()
    G = torch.zeros(fl.n, device=fl.dev)
    for t, (lr, g) in enumerate(zip(lrs, grads), 1):
        before, p = {k: v.clone() for k, v in fl.st.items()}, fl.params()
        G.copy_(g)
        fl.step(G, lr, t, args)
        want, want_p, aux = restate(fl, before, p, G, float(fl.sumsq), lr, t, args)
        compare_step(fl, fl.st, fl.params(), want, want_p, aux, acc)
    n8 = int(fl.bw.sum()) * len(lrs)
    for k in ("state1", "state2"):
        acc[k + "_differ_share"] = acc[k + "_differ"] / max(1, n8)
        if not acc[k + "_differ_share"] < 1e-4:
            acc["fail"].append(f"{k}: {acc[k + '_differ_share']:.2e} of the codes differ")
    acc["params_differ_share"] = acc["params_differ"] / max(1, acc["elements"])
    st, p = {k: torch.zeros_like(v) for k, v in fl.st.items()}, start.clone()
    for t, (lr, g) in enumerate(zip(lrs, grads), 1):
        st, p, _ = restate(fl, st, p, g, float((g.double() ** 2).sum()), lr, t, args)
    got = fl.params()
    acc["free_rel_l2"] = harness.rel_l2(got, p)
    acc["free_rel_l2_of_displacement"] = float((got.double() - p.double()).norm() / ((p.double() - start.double()).norm() + 1e-30))
    if not acc["free_rel_l2"] <= free_tol:
        acc["fail"].append(f"rel-L2 against the free-running restatement {acc['free_rel_l2']:.3e}")
    return acc


def kernel_flux_yaml():
    from prodigy_check import FlatLora, _flux_yaml_shapes
    fl_p = FlatLora(_flux_yaml_shapes(), 32, 11)
    fl = Flat(fl_p.members, fl_p.n, "cuda")
    lrs = cosine_lrs(ARGS["lr"])
    res = check_run(fl, [fl_p.grads(t, 5) for t in range(len(lrs))], lrs)
    res["fp32_path_elements"] = int((~fl.bw).sum())
    if any(bool(b[:, fl_p.r:].any()) for b in fl_p.bufs):
        res["fail"].append("B padding columns written")
    return res


def kernel_small_and_partial(dev="cuda"):
    import torch
    g = torch.Generator().manual_seed(3)
    rn = lambda *s: (torch.randn(*s, generator=g) * 0.05).bfloat16().to(dev)
    buf = torch.zeros(300, 64, dtype=torch.bfloat16, device=dev)
    buf[:, :16] = rn(300, 16)
    params = [rn(3, 1365), rn(16, 256), rn(8, 625), buf[:, :16]]
    members, off = [], 0
    for p in params:
        members.append((p, off))
        off += p.numel()
    fl = Flat(members, off, dev)
    zero_block = slice(members[1][1] + 768, members[1][1] + 1024)
    grads = []
    for t in range(6):
        gr = (torch.randn(off, generator=g) * 0.02).to(dev)
        gr[zero_block] = 0
        grads.append(gr)
    res = check_run(fl, grads, cosine_lrs(1e-2, 6, 2), dict(ARGS, lr=1e-2, weight_decay=0.01), free_tol=1e-2)
    s, so = fl.st, fl.offsets.tolist()
    if not (fl.bw[members[0][1]: members[1][1]].logical_not().all() and fl.bw[members[1][1]:].all()):
        res["fail"].append("4095 elements must take the fp32 path, 4096 and more the 8-bit one")
    if bool(s["state1"][: members[1][1]].any()) or not bool(s["s1_32"].any()):
        res["fail"].append("the fp32-path tensor must keep fp32 states and leave its codes alone")
    blk = so[1] + 3
    if float(s["absmax1"][blk]) != 0 or float(s["absmax2"][blk]) != 0:
        res["fail"].append("the zero-gradient block's absmax must be 0")
    if not (s["state1"][zero_block].eq(127).all() and s["state2"][zero_block].eq(0).all()):
        res["fail"].append("the zero-gradient block must hold the zero codes")
    nb = -(-5000 // 256)
    if fl.st["absmax1"][so[2]: so[2] + nb].eq(0).any():
        res["fail"].append("the partial last block of the 5000-element tensor was not updated")
    if bool(buf[:, 16:].any()):
        res["fail"].append("B padding columns written")
    return res


def repeat_bitwise():
    import torch
    from prodigy_check import FlatLora, _flux_yaml_shapes
    runs = []
    for _ in range(2):
        fl_p = FlatLora(_flux_yaml_shapes(), 32, 11)
        fl = Flat(fl_p.members, fl_p.n, "cuda")
        G = torch.zeros(fl.n, device="cuda")
        for t, lr in enumerate(cosine_lrs(ARGS["lr"], 4, 1), 1):
            G.copy_(fl_p.grads(t, 5))
            fl.step(G, lr, t)
        torch.cuda.synchronize()
        runs.append([fl.params()] + [fl.st[k] for k in sorted(fl.st)])
    same = [torch.equal(a.view(torch.uint8), b.view(torch.uint8)) for a, b in zip(*runs)]
    return dict(same=same, fail=[] if all(same) else ["two runs differ"])


def _step_case(family):
    import torch
    import bench
    import nf4_check
    from qflux_b200.optim import FusedLoraAdam8bit
    dev = torch.device("cuda", 0)
    torch.manual_seed(1234)
    if family == "qwen":
        cfg = dict(bench.CONFIGS["qwen_edit"], blocks=2)
        m = bench.build_model(dev, 2, cfg)
        name = "qwen_edit"
    else:
        cfg = dict(bench.CONFIGS["flux_kontext"])
        m = bench.build_flux(dev, cfg, 2 / 38)
        name = "flux_kontext"
    step = nf4_check._step(m, family)
    batch = nf4_check.device_batch(cfg, name)
    opt = FusedLoraAdam8bit(m, lr=ARGS["lr"], betas=ARGS["betas"], max_grad_norm=1.0)
    fl = Flat(opt._members, m.G32.numel(), dev)
    start = fl.params()
    grads, losses = [], []
    for _ in range(3):
        losses.append(float(step.train_step(batch, opt)))
        grads.append(m.G32.clone())
    torch.cuda.synchronize()
    st, p = {k: torch.zeros_like(v) for k, v in fl.st.items()}, start.clone()
    for t, g in enumerate(grads, 1):
        st, p, _ = restate(fl, st, p, g, float((g.double() ** 2).sum()), ARGS["lr"], t)
    got = fl.params()
    res = dict(family=family, losses=losses, lora_elements=fl.n, fail=[])
    res["rel_l2_of_displacement"] = float((got.double() - p.double()).norm() / ((p.double() - start.double()).norm() + 1e-30))
    n8 = max(1, int(fl.bw.sum()))
    res["codes_differ_share"] = [int((opt.state1 != st["state1"]).sum()) / n8, int((opt.state2 != st["state2"]).sum()) / n8]
    if not all(math.isfinite(l) for l in losses) or not bool(torch.isfinite(got.float()).all()):
        res["fail"].append("non-finite loss or parameters")
    if not res["rel_l2_of_displacement"] <= 1e-2:
        res["fail"].append(f"parameters {res['rel_l2_of_displacement']:.3e} of the displacement from the restatement")
    if not max(res["codes_differ_share"]) <= 1e-3:
        res["fail"].append(f"codes differ: {res['codes_differ_share']}")
    return res


CASES = dict(kernel_flux_yaml=kernel_flux_yaml, kernel_small_and_partial=kernel_small_and_partial, repeat_bitwise=repeat_bitwise,
             step_qwen=lambda: _step_case("qwen"), step_flux_yaml=lambda: _step_case("flux"))

if __name__ == "__main__":
    harness.main(CASES, os.path.abspath(__file__), "adam8bit_check.log")
