"""GPU check of qfx_gemm_bf16 against torch fp32 matmul (run under gpurun)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from harness import main, rel_l2, time_cuda  # noqa: E402

import torch  # noqa: E402


def _mk(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, device="cuda", generator=g) * scale).bfloat16()


def _gelu_grad(u):
    u = u.detach().float().requires_grad_(True)
    torch.nn.functional.gelu(u, approximate="tanh").sum().backward()
    return u.grad


def basic(trans_b, bn, M=300, N=768, K=256, bias=True, alpha=1.0):
    from qflux_b200 import lib
    A = _mk(M, K, seed=1)
    W = _mk(K, N, seed=2) if trans_b else _mk(N, K, seed=2)
    b = _mk(N, seed=3) if bias else None
    out = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    lib.gemm([lib.gemm_problem(A, W, out, bias=b)], N, K, trans_b=trans_b, alpha=alpha, block_n=bn)
    torch.cuda.synchronize()
    ref = alpha * (A.float() @ (W.float() if trans_b else W.float().t()))
    if bias:
        ref = ref + b.float()
    return dict(err=rel_l2(out.float(), ref))


def lora(trans_b, bn, M=520, N=768, K=512, kb2=1, groups=1):
    """acc = A.B(^T) + A2[:, slice].B2(^T) ; groups>1 => fused q|k|v (trans_b=0 only)."""
    from qflux_b200 import lib
    A = _mk(M, K, seed=1)
    W = _mk(K, N, seed=2) if trans_b else _mk(N, K, seed=2)
    r = 64 * kb2
    a2c = 0
    A2 = _mk(M, r * groups, seed=4)
    B2 = _mk(r, N, seed=5) if trans_b else _mk(N, r, seed=5)
    out = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    gn = N // groups if groups > 1 else 0
    lib.gemm([lib.gemm_problem(A, W, out, A2=A2, B2=B2, kb2=kb2, a2_col0=a2c)], N, K, trans_b=trans_b, lora_group_n=gn,
             block_n=bn)
    torch.cuda.synchronize()
    ref = A.float() @ (W.float() if trans_b else W.float().t())
    if trans_b:
        ref = ref + A2.float() @ B2.float()
    else:
        for g in range(groups):
            n0, n1 = g * (N // groups), (g + 1) * (N // groups)
            ref[:, n0:n1] += A2[:, g * r:(g + 1) * r].float() @ B2[n0:n1].float().t()
    return dict(err=rel_l2(out.float(), ref))


def epilogues(bn, M=384, N=512, K=256, Bsz=3):
    from qflux_b200 import lib
    A, W, b = _mk(M, K, seed=1), _mk(N, K, seed=2, scale=0.1), _mk(N, seed=3)
    res = {}
    # GELU
    out, u = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16), torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    lib.gemm([lib.gemm_problem(A, W, out, bias=b, out2=u)], N, K, epilogue=lib.EPI_GELU, block_n=bn)
    ref_u = A.float() @ W.float().t() + b.float()
    res["gelu_u"] = rel_l2(u.float(), ref_u)
    res["gelu"] = rel_l2(out.float(), torch.nn.functional.gelu(ref_u, approximate="tanh"))
    # RESID_GATE
    resid, gate = _mk(M, N, seed=6), _mk(Bsz, N, seed=7)
    out = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    lib.gemm([lib.gemm_problem(A, W, out, bias=b, resid=resid, gate=gate, rows_per_batch=M // Bsz)], N, K,
             epilogue=lib.EPI_RESID_GATE, block_n=bn)
    ref = resid.float() + gate.float().repeat_interleave(M // Bsz, 0) * ref_u
    res["resid_gate"] = rel_l2(out.float(), ref)
    # RESID_GATE with the optional second output (un-gated branch, kept when the gate's AdaLN linear carries LoRA)
    out_b, y = torch.zeros_like(out), torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    lib.gemm([lib.gemm_problem(A, W, out_b, bias=b, resid=resid, gate=gate, rows_per_batch=M // Bsz, out2=y)], N, K,
             epilogue=lib.EPI_RESID_GATE, block_n=bn)
    res["resid_gate_out2"] = max(rel_l2(y.float(), ref_u), rel_l2(out_b.float(), out.float()))
    # DGELU (trans_b)
    Wt = _mk(K, N, seed=8, scale=0.1)
    aux = _mk(M, N, seed=9)
    out = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    lib.gemm([lib.gemm_problem(A, Wt, out, aux=aux)], N, K, trans_b=True, epilogue=lib.EPI_DGELU, block_n=bn)
    ref = (A.float() @ Wt.float()) * _gelu_grad(aux)
    res["dgelu"] = rel_l2(out.float(), ref)
    torch.cuda.synchronize()
    res["err"] = max(res.values())
    return res


def grouped(trans_b, bn, N=768, K=512, M0=700, M1=130):
    from qflux_b200 import lib
    A0, A1 = _mk(M0, K, seed=1), _mk(M1, K, seed=2)
    W0 = _mk(K, N, seed=3) if trans_b else _mk(N, K, seed=3)
    W1 = _mk(K, N, seed=4) if trans_b else _mk(N, K, seed=4)
    A2 = _mk(M0, 64, seed=5)
    B2 = _mk(64, N, seed=6) if trans_b else _mk(N, 64, seed=6)
    o0 = torch.zeros(M0, N, device="cuda", dtype=torch.bfloat16)
    o1 = torch.zeros(M1, N, device="cuda", dtype=torch.bfloat16)
    lib.gemm([lib.gemm_problem(A0, W0, o0, A2=A2, B2=B2, kb2=1), lib.gemm_problem(A1, W1, o1)], N, K, trans_b=trans_b,
             block_n=bn)
    torch.cuda.synchronize()
    f = (lambda a, w: a.float() @ w.float()) if trans_b else (lambda a, w: a.float() @ w.float().t())
    r0 = f(A0, W0) + f(A2, B2)
    return dict(err=max(rel_l2(o0.float(), r0), rel_l2(o1.float(), f(A1, W1))))


def many(trans_b, bn, Ms=(700, 130, 256, 1, 385, 64), N=64, K=768, timing=False):
    """Up to QFX_MAX_PROBLEMS = 6 row groups in one launch (the U = s dY B projections of the three q|k|v slots of both streams of a LoRA
    backward): every problem has its own A, B and output, slices of wider buffers like the real call; one of them carries a LoRA k-block."""
    from qflux_b200 import lib
    wide = [_mk(M, 3 * K, seed=10 + i) for i, M in enumerate(Ms)]          # dY [M, 3*out]: problem i reads column slice i % 3
    A = [w[:, (i % 3) * K:(i % 3 + 1) * K] for i, w in enumerate(wide)]
    W = [(_mk(K, N, seed=30 + i, scale=0.1) if trans_b else _mk(N, K, seed=30 + i, scale=0.1)) for i in range(len(Ms))]
    outw = [torch.zeros(M, 3 * N, device="cuda", dtype=torch.bfloat16) for M in Ms]
    out = [o[:, (i % 3) * N:(i % 3 + 1) * N] for i, o in enumerate(outw)]
    A2, B2 = _mk(Ms[0], 64, seed=50), (_mk(64, N, seed=51) if trans_b else _mk(N, 64, seed=51))
    probs = [lib.gemm_problem(A[i], W[i], out[i], **(dict(A2=A2, B2=B2, kb2=1) if i == 0 else {})) for i in range(len(Ms))]
    lib.gemm(probs, N, K, trans_b=trans_b, alpha=0.5 if N == 64 else 1.0, block_n=bn)
    torch.cuda.synchronize()
    f = (lambda a, w: a.float() @ w.float()) if trans_b else (lambda a, w: a.float() @ w.float().t())
    alpha = 0.5 if N == 64 else 1.0
    errs = []
    for i in range(len(Ms)):
        ref = alpha * (f(A[i], W[i]) + (f(A2, B2) if i == 0 else 0))
        errs.append(rel_l2(out[i].float(), ref))
        others = torch.cat([outw[i][:, :(i % 3) * N], outw[i][:, (i % 3 + 1) * N:]], 1)
        assert float(others.abs().max()) == 0.0, "a problem wrote outside its column slice"
    res = dict(err=max(errs))
    if timing:  # six launches vs one, at the LoRA backward shape of the benchmark (image 8192 rows, text 1408 rows, out = 3072)
        Mi, Mt, Ko = 8192, 1408, 3072
        dY = [_mk(Mi, 3 * Ko, seed=1), _mk(Mt, 3 * Ko, seed=2)]
        Bp = [_mk(3 * Ko, 64, seed=3, scale=0.1), _mk(3 * Ko, 64, seed=4, scale=0.1)]
        U = [torch.zeros(Mi, 192, device="cuda", dtype=torch.bfloat16), torch.zeros(Mt, 192, device="cuda", dtype=torch.bfloat16)]
        pr = [lib.gemm_problem(dY[s][:, g * Ko:(g + 1) * Ko], Bp[s][g * Ko:(g + 1) * Ko], U[s][:, g * 64:(g + 1) * 64]) for s in range(2) for g in range(3)]
        flush = torch.empty(256 << 20, device="cuda", dtype=torch.uint8)
        res["one_launch_ms"] = time_cuda(lambda: lib.gemm(pr, 64, Ko, trans_b=True), flush=flush)
        res["six_launches_ms"] = time_cuda(lambda: [lib.gemm([q], 64, Ko, trans_b=True) for q in pr], flush=flush)
    return res


def attn_do(bn, H=2, Bsz=3, T=40, L=260, K=512, lora=True):
    """QFX_EPI_ATTN_DO: the out-projection dgrad writes dO head-major into dO_joint [B, H, S, 128] and delta = rowsum(dO * O) — checked
    against the plain dgrad (fp32 matmul, bf16-rounded) followed by the attn_delta semantics.  Two row groups (image: positions T.., text: 0..)."""
    from qflux_b200 import lib
    N, S = H * 128, T + L
    Mi, Mt = Bsz * L, Bsz * T
    dY = [_mk(Mi, K, seed=1), _mk(Mt, K, seed=2)]
    W = [_mk(K, N, seed=3, scale=0.1), _mk(K, N, seed=4, scale=0.1)]
    O = [_mk(Mi, N, seed=5), _mk(Mt, N, seed=6)]
    A2, B2 = _mk(Mi, 64, seed=7), _mk(64, N, seed=8, scale=0.1)
    dOj = torch.full((Bsz, H, S, 128), 9.0, device="cuda", dtype=torch.bfloat16)
    delta = torch.full((Bsz, H, S), 9.0, device="cuda")
    tok = [torch.zeros(Mi, N, device="cuda", dtype=torch.bfloat16), None]
    probs = [lib.gemm_problem(dY[s], W[s], dOj, aux=O[s], delta=delta, rows_per_batch=(L, T)[s], s_offset=(T, 0)[s], out2=tok[s],
                              **(dict(A2=A2, B2=B2, kb2=1) if (lora and s == 0) else {})) for s in range(2)]
    lib.gemm(probs, N, K, trans_b=True, epilogue=lib.EPI_ATTN_DO, block_n=bn)
    torch.cuda.synchronize()
    ref = [dY[s].float() @ W[s].float() + ((A2.float() @ B2.float()) if (lora and s == 0) else 0) for s in range(2)]
    g = [r.bfloat16() for r in ref]
    want_j = torch.cat([g[1].view(Bsz, T, H, 128), g[0].view(Bsz, L, H, 128)], 1).permute(0, 2, 1, 3).float()
    want_d = torch.cat([(g[1].float() * O[1].float()).view(Bsz, T, H, 128).sum(-1), (g[0].float() * O[0].float()).view(Bsz, L, H, 128).sum(-1)], 1).permute(0, 2, 1)
    res = dict(dOj=rel_l2(dOj.float(), want_j), delta=rel_l2(delta, want_d), token_major=rel_l2(tok[0].float(), g[0].float()))
    res["err"] = max(res.values())
    return res


def perf(trans_b, bn, M0=8192, M1=1408, N=3072, K=3072):
    from qflux_b200 import lib
    A0, A1 = _mk(M0, K, seed=1), _mk(M1, K, seed=2)
    W0 = _mk(K, N, seed=3, scale=0.02) if trans_b else _mk(N, K, seed=3, scale=0.02)
    W1 = _mk(K, N, seed=4, scale=0.02) if trans_b else _mk(N, K, seed=4, scale=0.02)
    o0 = torch.zeros(M0, N, device="cuda", dtype=torch.bfloat16)
    o1 = torch.zeros(M1, N, device="cuda", dtype=torch.bfloat16)
    probs = [lib.gemm_problem(A0, W0, o0), lib.gemm_problem(A1, W1, o1)]
    flush = torch.empty(256 << 20, device="cuda", dtype=torch.uint8)
    ms = time_cuda(lambda: lib.gemm(probs, N, K, trans_b=trans_b, block_n=bn), flush=flush)
    fl = 2.0 * (M0 + M1) * N * K
    f = (lambda a, w: a @ w) if trans_b else (lambda a, w: a @ w.t())
    ms_t = time_cuda(lambda: (f(A0, W0), f(A1, W1)), flush=flush)
    err = rel_l2(o0.float(), f(A0.float(), W0.float()))
    return dict(ms=round(ms, 4), tflops=round(fl / ms / 1e9, 1), torch_ms=round(ms_t, 4), torch_tflops=round(fl / ms_t / 1e9, 1),
                err=err)


def ragged(bn, trans_b=False, R=1600, valid=(1600, 400, 1024, 900), N=768, K=512, perf=False):
    """Ragged row groups (qfx_gemm_problem.row_tiles): a grouped launch whose first problem is a pad-to-max image stream (sample b owns rows
    [b*R, (b+1)*R), valid[b] of them real) and whose second is a dense text stream.  Rows inside the computed 256-row bands must equal the
    dense result, every other row of the outputs must be exactly zero; covers BIAS, GELU (two outputs) and RESID_GATE / DGELU."""
    from qflux_b200 import lib
    M0, M1, Bsz = R * len(valid), 300, len(valid)
    plan = lib.RowBands.plan(list(valid), R)
    bands = lib.RowBands(plan[0], plan[1], "cuda")
    live = torch.zeros(M0, dtype=torch.bool, device="cuda")
    for t in bands.host_tiles:
        live[t:t + 256] = True
    for lo, hi in bands.host_dead:
        assert not live[lo:hi].any()
    A = [_mk(M0, K, seed=1), _mk(M1, K, seed=2)]
    W = [(_mk(K, N, seed=3 + i, scale=0.1) if trans_b else _mk(N, K, seed=3 + i, scale=0.1)) for i in range(2)]
    b = [None, None] if trans_b else [_mk(N, seed=5), _mk(N, seed=6)]
    mm = lambda i: A[i].float() @ (W[i].float() if trans_b else W[i].float().t()) + (0 if trans_b else b[i].float())
    res, worst = {}, 0.0

    def run(epi, **extra):
        outs = [torch.full((M, N), 7.0, device="cuda", dtype=torch.bfloat16) for M in (M0, M1)]
        out2 = [torch.full((M, N), 7.0, device="cuda", dtype=torch.bfloat16) for M in (M0, M1)] if epi in (lib.EPI_GELU, lib.EPI_RESID_GATE) else [None, None]
        probs = [lib.gemm_problem(A[i], W[i], outs[i], bias=b[i], out2=out2[i], row_bands=bands if i == 0 else None,
                                  **{k: v[i] for k, v in extra.items()}) for i in range(2)]
        lib.gemm(probs, N, K, trans_b=trans_b, epilogue=epi, block_n=bn)
        torch.cuda.synchronize()
        return outs, out2

    def check(name, got, ref):
        nonlocal worst
        e_live = rel_l2(got[0][live].float(), ref[0][live])
        dead_max = float(got[0][~live].float().abs().max()) if (~live).any() else 0.0
        e_txt = rel_l2(got[1].float(), ref[1])
        res[name] = (round(e_live, 6), dead_max, round(e_txt, 6))
        worst = max(worst, e_live, e_txt, 1.0 if dead_max != 0.0 else 0.0)

    if not trans_b:
        o, _ = run(lib.EPI_BIAS)
        check("bias", o, [mm(0), mm(1)])
        o, u = run(lib.EPI_GELU)
        check("gelu", o, [torch.nn.functional.gelu(mm(i), approximate="tanh") for i in range(2)])
        check("gelu_u", u, [mm(0), mm(1)])
        resid = [_mk(M0, N, seed=8), _mk(M1, N, seed=9)]
        gate = [_mk(Bsz, N, seed=10), _mk(3, N, seed=11)]
        o, y = run(lib.EPI_RESID_GATE, resid=resid, gate=gate, rows_per_batch=[R, M1 // 3])
        check("resid_gate", o, [resid[i].float() + gate[i].float().repeat_interleave([R, M1 // 3][i], 0) * mm(i) for i in range(2)])
        check("resid_gate_y", y, [mm(0), mm(1)])
    else:
        o, _ = run(lib.EPI_BIAS)
        check("dgrad", o, [mm(0), mm(1)])
        aux = [_mk(M0, N, seed=12), _mk(M1, N, seed=13)]
        o, _ = run(lib.EPI_DGELU, aux=aux)
        check("dgelu", o, [mm(i) * _gelu_grad(aux[i]) for i in range(2)])
    out = dict(err=worst, cases=res, bands=bands.n, dead_ranges=bands.host_dead)
    if perf:  # the benchmark's multi-resolution mix at the MLP-up shape: ragged vs dense launch
        Rp, vp, Np, Kp = 1600, (1600, 400, 1024, 1024), 12288, 3072
        plan = lib.RowBands.plan(list(vp), Rp)
        bp = lib.RowBands(plan[0], plan[1], "cuda")
        Ab, Wb = _mk(4 * Rp, Kp, seed=1), _mk(Np, Kp, seed=2, scale=0.05)
        ob, ub = torch.empty(4 * Rp, Np, device="cuda", dtype=torch.bfloat16), torch.empty(4 * Rp, Np, device="cuda", dtype=torch.bfloat16)
        flush = torch.empty(256 << 20, device="cuda", dtype=torch.uint8)
        for nm, rb in (("dense_ms", None), ("ragged_ms", bp)):
            pr = [lib.gemm_problem(Ab, Wb, ob, bias=None, out2=ub, row_bands=rb)]
            out[nm] = time_cuda(lambda: lib.gemm(pr, Np, Kp, epilogue=lib.EPI_GELU), iters=10, flush=flush)
        out["live_fraction"] = bp.n * 256 / (4 * Rp)
    return out


CASES = {}
CASES["attn_do_bn256"] = lambda: attn_do(256)
CASES["attn_do_bn128_h3"] = lambda: attn_do(0, H=3)
CASES["cta2_attn_do"] = lambda: attn_do(1256, H=4, K=1024)
CASES["cta2_attn_do_splitk"] = lambda: attn_do(1256, H=16, Bsz=4, T=40, L=600, K=4096)
CASES["many6_nn_bn64"] = lambda: many(True, 64)
CASES["many6_nt_bn64"] = lambda: many(False, 64)
CASES["many5_nt_bn192"] = lambda: many(False, 192, Ms=(300, 130, 256, 129, 64), N=192)
CASES["cta2_many6_nn"] = lambda: many(True, 1256, N=256, K=512)
CASES["cta2_many4_nt_splitk"] = lambda: many(False, 1256, Ms=(2304, 256, 130, 700), N=2048, K=4096)
CASES["many6_timing"] = lambda: many(True, 64, timing=True)
CASES["ragged_nt_bn256"] = lambda: ragged(256)
CASES["ragged_nt_bn128"] = lambda: ragged(128)
CASES["ragged_nn_bn192"] = lambda: ragged(192, trans_b=True)
CASES["cta2_ragged_nt"] = lambda: ragged(1256)
CASES["cta2_ragged_nn"] = lambda: ragged(1256, trans_b=True)
CASES["cta2_ragged_nt_splitk"] = lambda: ragged(1256, N=2048, K=4096)
CASES["cta2_ragged_perf"] = lambda: ragged(1256, perf=True)
for bn in (64, 128, 192, 256):
    CASES[f"basic_nt_bn{bn}"] = (lambda bn=bn: basic(False, bn))
    CASES[f"basic_nn_bn{bn}"] = (lambda bn=bn: basic(True, bn))
for bn in (1128, 1256):
    CASES[f"cta2_basic_nt_bn{bn}"] = (lambda bn=bn: basic(False, bn, M=700, N=768, K=512))
    CASES[f"cta2_basic_nn_bn{bn}"] = (lambda bn=bn: basic(True, bn, M=700, N=768, K=512))
    CASES[f"cta2_lora_nt_bn{bn}"] = (lambda bn=bn: lora(False, bn, N=768, groups=3))
    CASES[f"cta2_lora_nn_bn{bn}"] = (lambda bn=bn: lora(True, bn, kb2=3))
CASES["cta2_epilogues"] = lambda: epilogues(1256)
# *_splitk cases (names kept): long K (4096-4608, 64-72 k-blocks per tile, many turns of the TMA ring); the sm_90a kernel has no split-K
CASES["cta2_splitk_epilogues"] = lambda: epilogues(1256, M=2560, N=2048, K=4096, Bsz=4)
CASES["cta2_splitk_lora_nt"] = lambda: lora(False, 1256, M=2560, N=2048, K=4096)
CASES["cta2_splitk_lora_nn"] = lambda: lora(True, 1256, M=2560, N=2048, K=4096, kb2=3)
CASES["cta2_splitk_grouped_nn"] = lambda: grouped(True, 1256, K=4608, N=2560, M0=1900, M1=300)
CASES["cta2_grouped_nt"] = lambda: grouped(False, 1256)
CASES["cta2_grouped_nn"] = lambda: grouped(True, 1128)
CASES["cta2_perf_nt"] = lambda: perf(False, 1256)
CASES["cta2_perf_nn"] = lambda: perf(True, 1256)
CASES["cta2_perf_nt_mlp_up"] = lambda: perf(False, 1256, N=12288, K=3072)
CASES["cta2_perf_nt_mlp_down"] = lambda: perf(False, 1256, N=3072, K=12288)
CASES["cta2_perf_nn_mlp_down"] = lambda: perf(True, 1256, N=12288, K=3072)
CASES["cta2_perf_nt_bn128"] = lambda: perf(False, 1128)
CASES["cta2_perf_nn_bn128_k9216"] = lambda: perf(True, 1128, N=3072, K=9216)
CASES["cta2_perf_nn_bn256_k9216"] = lambda: perf(True, 1256, N=3072, K=9216)
CASES["cta2_perf_nt_bn128_down"] = lambda: perf(False, 1128, N=3072, K=12288)
CASES["basic_nt_alpha_nobias"] = lambda: basic(False, 0, M=128, N=64, K=64, bias=False, alpha=0.5)
CASES["basic_nt_big"] = lambda: basic(False, 0, M=2400, N=3072, K=3072)
CASES["basic_nn_big"] = lambda: basic(True, 0, M=2400, N=3072, K=12288)
for bn in (128, 256):
    CASES[f"lora_nt_bn{bn}"] = (lambda bn=bn: lora(False, bn))
    CASES[f"lora_nn_bn{bn}"] = (lambda bn=bn: lora(True, bn))
CASES["lora_nt_groups3"] = lambda: lora(False, 128, N=768, groups=3)
CASES["lora_nt_kb2"] = lambda: lora(False, 192, kb2=2)
CASES["lora_nn_kb3"] = lambda: lora(True, 192, kb2=3)
CASES["epilogues_bn128"] = lambda: epilogues(128)
CASES["epilogues_bn256"] = lambda: epilogues(256)
CASES["grouped_nt"] = lambda: grouped(False, 256)
CASES["grouped_nn"] = lambda: grouped(True, 192)
for bn in (128, 192, 256):
    CASES[f"perf_nt_bn{bn}"] = (lambda bn=bn: perf(False, bn))
    CASES[f"perf_nn_bn{bn}"] = (lambda bn=bn: perf(True, bn))
CASES["perf_nt_mlp_up"] = lambda: perf(False, 256, N=12288, K=3072)
CASES["perf_nt_mlp_down"] = lambda: perf(False, 256, N=3072, K=12288)
CASES["perf_nn_mlp_down"] = lambda: perf(True, 256, N=12288, K=3072)

if __name__ == "__main__":
    main(CASES, os.path.abspath(__file__), "gemm_check.log")
