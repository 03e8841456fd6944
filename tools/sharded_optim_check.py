"""GPU check of the sharded optimizer's kernels (qfx.h "slice forms", qfx_lora_pack / unpack), one case per call:

  python tools/sharded_optim_check.py pack|sumsq|adamw|adam8bit|prodigy

The tables have the factor shapes of the block Linears of FLUX-Kontext with the YAML targets at r = 32: A [32, d_in] and B [d_out, 32]
with row stride 64 (the padded factor buffers), 171.8 M elements (the embedders' 0.1 M left out).  Slices come from
sharding.SlicePlan at world 3, so they start and end inside tensors.  Each slice form, run for every slice of the plan, must give the bits of the replicated entry point on the same gradient
(the clip inactive); pack must equal an indexed copy, unpack must restore the weights and write nothing else; the sum of squares must
match fp64.  Exit code 0 when every check holds."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.join(os.path.dirname(HERE), "qwen-image-finetune_b200")]

from qflux_b200 import lib  # noqa: E402
from qflux_b200.sharding import SlicePlan  # noqa: E402

D, R, RP = 3072, 32, 64
FLUX_YAML_R32 = 171_935_744


def members():
    """Factor pairs of FLUX-Kontext's YAML targets (19 double blocks, 38 single blocks) at r = 32, in registration order."""
    shapes = []
    for _ in range(19):
        shapes += [(D, D)] * 8 + [(D, 6 * D)] * 2 + [(D, 4 * D), (4 * D, D)] * 2
    for _ in range(38):
        shapes += [(D, D)] * 3 + [(D, 3 * D), (D, 4 * D), (5 * D, D)]
    out, off = [], 0
    for d_in, d_out in shapes:
        a = torch.randn(R, d_in, device="cuda").bfloat16()
        bpad = torch.zeros(d_out, RP, device="cuda", dtype=torch.bfloat16)
        bpad[:, :R] = torch.randn(d_out, R, device="cuda").bfloat16()
        b = bpad[:, :R]
        out += [(a, off), (b, off + a.numel())]
        off += a.numel() + b.numel()
    return out, off


def flat_weights(ms, n):
    w = torch.zeros(n, device="cuda", dtype=torch.bfloat16)
    for p, off in ms:
        w[off: off + p.numel()] = p.reshape(-1)
    return w


def bits(a, b):
    return torch.equal(a.reshape(-1).view(torch.uint8), b.reshape(-1).view(torch.uint8))


def setup(world=3):
    torch.manual_seed(0)
    ms, n = members()
    plan = SlicePlan(ms, n, world)
    tables = lib.adamw_tables(plan.members, "cuda")
    return ms, n, plan, tables


def case_pack():
    ms, n, plan, tables = setup()
    w = flat_weights(ms, n)
    ok = True
    for q in range(plan.world):
        lo, hi = plan.bounds[q]
        for a, b in ((lo, hi), (lo + 7, hi - 5), (lo + 1_000_003, lo + 3_000_001)):
            flat = torch.full((b - a + 16,), 3.0, device="cuda", dtype=torch.bfloat16)
            lib.lora_pack(tables, plan.chunks_in(q, a, b), a, b, flat[8:])
            ok &= bits(flat[8: 8 + b - a], w[a:b]) and bool((flat[:8] == 3).all() and (flat[8 + b - a:] == 3).all())
    before = [p.clone() for p, _ in ms]
    sentinel = [p._base.clone() if p._base is not None else None for p, _ in ms]
    for p, _ in ms:
        p.zero_()
    for q in range(plan.world):
        lo, hi = plan.bounds[q]
        lib.lora_unpack(tables, plan.chunk_ranges[q], lo, hi, w[lo:hi].contiguous())
    ok &= all(bits(p, b) for (p, _), b in zip(ms, before))
    ok &= all(s is None or bits(p._base[:, R:], s[:, R:]) for (p, _), s in zip(ms, sentinel))  # the padding columns stay as they were
    torch.cuda.synchronize()
    print("pack/unpack", "ok" if ok else "MISMATCH", "elements", n)
    return ok


def case_sumsq():
    x = torch.randn(FLUX_YAML_R32 // 3 + 11, device="cuda")
    out = torch.zeros(1, device="cuda")
    lib.sumsq_det(x[5:], 0.5, out, scratch=torch.zeros(lib.DET_NORM_PARTIALS, device="cuda"))
    ref = float(((x[5:].double() * 0.5) ** 2).sum())
    rel = abs(float(out) - ref) / ref
    print("sumsq rel", rel)
    return rel < 1e-6


def _grad(n):
    return torch.randn(n, device="cuda") * 1e-3


def case_adamw():
    ms, n, plan, tables = setup()
    g, start = _grad(n), [p.clone() for p, _ in ms]
    m, v, ss = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda"), torch.zeros(1, device="cuda")
    lib.fused_adamw_det(tables, g, m, v, ss, 0.5, 1e9, 1e-3, 0.9, 0.999, 1e-8, 1e-2, 1,
                        scratch=torch.zeros(lib.DET_NORM_PARTIALS, device="cuda"))
    ref_w, ref_m, ref_v = flat_weights(ms, n), m, v
    for (p, _), s in zip(ms, start):
        p.copy_(s)
    ok = True
    for q in range(plan.world):
        lo, hi = plan.bounds[q]
        mq, vq = torch.zeros(hi - lo, device="cuda"), torch.zeros(hi - lo, device="cuda")
        lib.fused_adamw_slice(tables, plan.chunk_ranges[q], lo, g, mq, vq, ss, 0.5, 1e9, 1e-3, 0.9, 0.999, 1e-8, 1e-2, 1)
        ok &= bits(mq, ref_m[lo:hi]) and bits(vq, ref_v[lo:hi])
    ok &= bits(flat_weights(ms, n), ref_w)
    print("adamw slices", "ok" if ok else "MISMATCH")
    return ok


def case_adam8bit():
    ms, n, plan, tables = setup()
    g, start = _grad(n), [p.clone() for p, _ in ms]
    offs, n_abs, n_small = lib.adam8bit_layout(plan.members, 4096)
    so = torch.tensor(offs, dtype=torch.int64, device="cuda")
    q1, q2 = lib.dynamic_map(True).cuda(), lib.dynamic_map(False).cuda()
    mk = lambda k, dt=torch.float32: torch.zeros(max(1, k), device="cuda", dtype=dt)
    st = [mk(n, torch.uint8), mk(n, torch.uint8), mk(n_abs), mk(n_abs), mk(n_small), mk(n_small)]
    ss = torch.zeros(1, device="cuda")
    lib.fused_adam8bit(tables, so, g, *st, q1, q2, ss, torch.zeros(lib.DET_NORM_PARTIALS, device="cuda"), 0.5, 1e9, 1e-3, 0.9, 0.999,
                       1e-8, 1e-2, 1, 4096)
    ref_w = flat_weights(ms, n)
    for (p, _), s in zip(ms, start):
        p.copy_(s)
    ok = True
    st2 = [mk(n, torch.uint8), mk(n, torch.uint8), mk(n_abs), mk(n_abs), mk(n_small), mk(n_small)]
    for q in range(plan.world):
        lo, hi = plan.bounds[q]
        # the slice's codes at index fi - lo; absmax / fp32 states in the whole arrays (offsets unchanged)
        lib.fused_adam8bit_slice(tables, plan.chunk_ranges[q], lo, so, g, st2[0][lo:hi], st2[1][lo:hi], *st2[2:], q1, q2, ss, 0.5, 1e9,
                                 1e-3, 0.9, 0.999, 1e-8, 1e-2, 1, 4096)
    ok &= all(bits(a, b) for a, b in zip(st, st2)) and bits(flat_weights(ms, n), ref_w)
    print("adam8bit slices", "ok" if ok else "MISMATCH")
    return ok


def case_prodigy():
    ms, n, plan, tables = setup()
    g, start = _grad(n), [p.clone() for p, _ in ms]
    p0 = flat_weights(ms, n)
    sc0 = torch.zeros(lib.PRODIGY_SCALARS, device="cuda", dtype=torch.float64)
    sc0[lib.PRODIGY_D] = sc0[lib.PRODIGY_D_MAX] = 1e-6
    for p, _ in ms:  # move the weights off p0 so the dot product is not zero
        p.add_(torch.randn_like(p) * 1e-2)
    start = [p.clone() for p, _ in ms]
    args = (1.0, 0.9, 0.999, 0.999 ** 0.5)
    ref = dict(m=torch.zeros(n, device="cuda"), v=torch.zeros(n, device="cuda"), s=torch.zeros(n, device="cuda"), sc=sc0.clone())
    ss = torch.zeros(1, device="cuda")
    lib.fused_prodigy(tables, g, ref["m"], ref["v"], ref["s"], p0, ref["sc"], ss,
                      torch.zeros(lib.prodigy_scratch_floats(tables), device="cuda"), 0.5, 1e9, *args, 1e-8, 1e-2, True, False, False,
                      1e-6, 1.0, float("inf"))
    ref_w = flat_weights(ms, n)
    for (p, _), s in zip(ms, start):
        p.copy_(s)
    sc = sc0.clone()
    part = torch.zeros(len(plan.chunks), 2, device="cuda", dtype=torch.float64)
    bufs = []
    for q in range(plan.world):
        lo, hi = plan.bounds[q]
        b = [torch.zeros(hi - lo, device="cuda") for _ in range(3)]
        lib.prodigy_slice_partials(tables, plan.chunk_ranges[q], lo, g, *b, p0[lo:hi].contiguous(), sc, ss, part, 0.5, 1e9, *args, 1e-2,
                                   True, False, False, 1e-6)
        bufs.append(b)
    table = torch.empty_like(part).index_copy_(0, torch.tensor(plan.table_chunk, device="cuda"), part)  # members are in order here
    for q in range(plan.world):
        lo, hi = plan.bounds[q]
        s_q = sc.clone()
        lib.prodigy_slice_update(tables, plan.chunk_ranges[q], lo, n, bufs[q][0], bufs[q][1], s_q, table, *args, 1e-8, 1e-2, True, False,
                                 1e-6, 1.0, float("inf"))
    ok = bits(s_q, ref["sc"]) and bits(flat_weights(ms, n), ref_w)
    for k, i in (("m", 0), ("v", 1), ("s", 2)):
        ok &= bits(torch.cat([b[i] for b in bufs]), ref[k])
    print("prodigy slices", "ok" if ok else "MISMATCH", "d", float(s_q[lib.PRODIGY_D]), float(ref["sc"][lib.PRODIGY_D]))
    return ok


if __name__ == "__main__":
    ok = globals()["case_" + sys.argv[1]]()
    sys.exit(0 if ok else 1)
