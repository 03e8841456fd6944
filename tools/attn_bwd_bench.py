"""Stand-alone timing of the joint attention backward at the benchmark's shape (H = 24, S = 352 + 2048 = 2400, head_dim 128):

    python tools/attn_bwd_bench.py                      this tree, B = 1 and B = 4
    python tools/attn_bwd_bench.py --ab OTHER_TREE      this tree and another checkout of the project, alternating in
                                                        subprocesses (ROUNDS rounds of: other, this), medians per tree

Timed per launch with CUDA events, the L2 flushed before each launch (as bench._time_kernel does):
  atomic   qfx_attn_bwd as the training step runs it: the caller's zero fill of the fp32 dQ accumulator, then the kernel
  det      qfx_attn_bwd_det (dK / dV by attn_bwd_kernel<false>, dQ by attn_bwd_dq_kernel), its dQ zero fill included
B = 1 runs the flagship's full prompt (txt_len 352), B = 4 a 40-token prompt (one 128-key tile fully masked, as in
tools/determinism_bench.py).  TFLOP/s counts the dense products from the shapes: 5 (S, dP, dV, dK, dQ) x 2 B H S^2 128 for
the atomic path, 7 for the deterministic one (S and dP are recomputed for dQ).  The card name and power limit are read in the
same process.
"""
import json
import os
import statistics
import subprocess
import sys

ROUNDS, ITERS = 5, 30


def _gpu():
    import torch
    try:
        pl = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the number is still valid; say why the power limit is missing
        pl = f"unavailable ({type(e).__name__})"
    return dict(gpu=torch.cuda.get_device_name(), power_limit=pl)


def measure(tree):
    """median ms per launch of both paths at B = 1 and B = 4, with the package of `tree`"""
    sys.path[:0] = [tree, os.path.join(tree, "qwen-image-finetune_b200")]
    import torch
    from qflux_b200 import lib
    assert os.path.dirname(os.path.abspath(lib.__file__)).startswith(os.path.abspath(tree))
    H, S, T = 24, 2400, 352
    flush = torch.empty(256 << 20, device="cuda", dtype=torch.uint8)
    out = {}
    for B, txt in ((1, T), (4, 40)):
        g = torch.Generator().manual_seed(B)
        Q, K, V, dO = (torch.randn(B, H, S, 128, generator=g).bfloat16().cuda() for _ in range(4))
        txt_len = torch.full((B,), txt, dtype=torch.int32, device="cuda")
        ot = torch.empty(B * T, H * 128, device="cuda", dtype=torch.bfloat16)
        oi = torch.empty(B * (S - T), H * 128, device="cuda", dtype=torch.bfloat16)
        lse = torch.empty(B, H, S, device="cuda")
        lib.attn_fwd(Q, K, V, ot, oi, T, lse, txt_len=txt_len)
        delta = (torch.randn(B, H, S, generator=g) * 0.1).cuda()
        dQ, dK, dV = torch.empty(B, H, S, 128, device="cuda"), torch.empty_like(Q), torch.empty_like(Q)
        for name, fn in (("atomic", lib.attn_bwd), ("det", lib.attn_bwd_det)):
            def run(fn=fn):
                dQ.zero_()
                fn(Q, K, V, dO, lse, delta, dQ, dK, dV, txt_len=txt_len, split=T)
            for _ in range(3):
                run()
            ts = []
            for _ in range(ITERS):
                flush.zero_()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run()
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            ms = statistics.median(ts)
            flop = (5 if name == "atomic" else 7) * 2 * B * H * S * S * 128
            out[f"{name}_B{B}"] = dict(ms=round(ms, 4), tflops=round(flop / ms / 1e9, 1))
    return dict(out, **_gpu())


def _one(tree):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", tree], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(r.stdout + r.stderr)
    return json.loads(r.stdout.strip().splitlines()[-1])


if __name__ == "__main__":
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if len(sys.argv) == 3 and sys.argv[1] == "--one":
        print(json.dumps(measure(sys.argv[2])))
    elif len(sys.argv) == 3 and sys.argv[1] == "--ab":
        trees = dict(base=os.path.abspath(sys.argv[2]), new=here)
        runs = {k: [] for k in trees}
        for _ in range(ROUNDS):
            for k, t in trees.items():
                runs[k].append(_one(t))
        keys = [k for k in runs["new"][0] if k.endswith(("_B1", "_B4"))]
        res = {}
        for k in keys:
            b = [r[k]["ms"] for r in runs["base"]]
            n = [r[k]["ms"] for r in runs["new"]]
            res[k] = dict(base_ms=statistics.median(b), new_ms=statistics.median(n), base_range=[min(b), max(b)],
                          new_range=[min(n), max(n)], speedup=round(statistics.median(b) / statistics.median(n), 3),
                          base_tflops=round(runs["base"][0][k]["tflops"] * runs["base"][0][k]["ms"] / statistics.median(b), 1),
                          new_tflops=round(runs["new"][0][k]["tflops"] * runs["new"][0][k]["ms"] / statistics.median(n), 1))
        res.update(gpu=runs["new"][-1]["gpu"], power_limit=runs["new"][-1]["power_limit"])
        print(json.dumps(res))
    else:
        print(json.dumps(measure(here)))
