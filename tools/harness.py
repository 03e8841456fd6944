"""Tiny GPU-check harness: every case runs in its own subprocess (a device trap must not poison the next case)."""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "qwen-image-finetune_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)


def rel_l2(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def time_cuda(fn, iters=20, warmup=3, flush=None):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def main(cases: dict, script: str, out_name: str, timeout: float = 300):
    if len(sys.argv) >= 3 and sys.argv[1] == "--case":
        res = cases[sys.argv[2]]()
        print("RESULT " + json.dumps(res))
        return
    only = sys.argv[1:] or list(cases)
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    log = open(os.path.join(ROOT, "gpurun_out", out_name), "a")
    ok_all = True
    for name in only:
        t0 = time.time()
        try:
            r = subprocess.run([sys.executable, script, "--case", name], capture_output=True, text=True, timeout=timeout)
            out = r.stdout + r.stderr
            res = [l for l in r.stdout.splitlines() if l.startswith("RESULT ")]
            status = "ok" if (r.returncode == 0 and res) else f"FAIL rc={r.returncode}"
            tail = res[-1][7:] if res else " | ".join(out.strip().splitlines()[-4:])[-700:]
        except subprocess.TimeoutExpired:
            status, tail = "TIMEOUT", ""
        ok_all &= status == "ok"
        line = f"[{status}] {name} ({time.time() - t0:.1f}s) {tail}"
        print(line, flush=True)
        log.write(line + "\n")
        log.flush()
    sys.exit(0 if ok_all else 1)
