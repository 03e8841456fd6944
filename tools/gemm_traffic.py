"""Time the step's big grouped GEMMs stand-alone (CUDA events, L2 flushed) — run it under `ncu --metrics dram__bytes_read.sum,
dram__bytes_write.sum,gpu__time_duration.sum` to get the DRAM traffic per launch (tools/ncu_traffic.py turns the csv into
a DRAM-traffic capture).  Shapes: Qwen-Image-Edit B=4 (8192 image + 1408 text rows)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from harness import ROOT, time_cuda  # noqa: F401,E402
import torch  # noqa: E402
from qflux_b200 import lib  # noqa: E402

dev = "cuda"
Mi, Mt, D = 8192, 1408, 3072
flush = torch.empty(256 << 20, device=dev, dtype=torch.uint8)
rn = lambda *s: (torch.randn(*s, device=dev) * 0.5).bfloat16()


def case(name, N, K, epi, trans_b=False):
    A = [rn(Mi, K), rn(Mt, K)]
    W = [rn(K, N) * 0.04 if trans_b else rn(N, K) * 0.04 for _ in range(2)]
    out = [torch.empty(Mi, N, device=dev, dtype=torch.bfloat16), torch.empty(Mt, N, device=dev, dtype=torch.bfloat16)]
    kw = [dict(), dict()]
    if epi == lib.EPI_GELU:
        kw = [dict(out2=torch.empty_like(o), bias=torch.zeros(N, device=dev, dtype=torch.bfloat16)) for o in out]
    elif epi == lib.EPI_DGELU:
        kw = [dict(aux=rn(*o.shape)) for o in out]
    elif epi == lib.EPI_RESID_GATE:
        g = rn(4, N)
        kw = [dict(resid=rn(*o.shape), gate=g, rows_per_batch=o.shape[0] // 4, bias=torch.zeros(N, device=dev, dtype=torch.bfloat16)) for o in out]
    elif epi == lib.EPI_BIAS and not trans_b:
        kw = [dict(bias=torch.zeros(N, device=dev, dtype=torch.bfloat16)) for o in out]
    probs = [lib.gemm_problem(A[i], W[i], out[i], **kw[i]) for i in range(2)]
    ms = time_cuda(lambda: lib.gemm(probs, N, K, trans_b=trans_b, epilogue=epi), iters=10, flush=flush)
    fl = 2.0 * (Mi + Mt) * N * K
    print(f"{name:28s} N={N:6d} K={K:6d} {ms:8.4f} ms {fl / ms / 1e9:8.1f} TFLOP/s", flush=True)


case("qkv   (BIAS)", 3 * D, D, lib.EPI_BIAS)
case("out   (RESID_GATE)", D, D, lib.EPI_RESID_GATE)
case("up    (GELU, 2 outputs)", 4 * D, D, lib.EPI_GELU)
case("down  (RESID_GATE)", D, 4 * D, lib.EPI_RESID_GATE)
case("d_down (dgrad DGELU)", 4 * D, D, lib.EPI_DGELU, trans_b=True)
case("d_up   (dgrad BIAS)", D, 4 * D, lib.EPI_BIAS, trans_b=True)
case("d_qkv  (dgrad BIAS)", D, 3 * D, lib.EPI_BIAS, trans_b=True)
