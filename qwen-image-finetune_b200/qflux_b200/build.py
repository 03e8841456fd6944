"""In-tree build of libqfx_b200.so:  nvcc -gencode arch=compute_90a,code=sm_90a  (cross-compiles without a GPU)."""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "csrc")
ROOT = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, "libqfx_b200.so")
OBJ = os.path.join(CSRC, "_obj")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC",
         "--use_fast_math", "-I", os.path.join(ROOT, "include")]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _headers_mtime():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(ROOT, "include", "qfx.h"))
    return max(os.path.getmtime(h) for h in hs)


def build_library(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    hm = _headers_mtime()
    jobs = []
    for src in _sources():
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src[:-3] + ".o")
        if force or not os.path.exists(o) or os.path.getmtime(o) < max(os.path.getmtime(s), hm):
            jobs.append((s, o))

    def cc(job):
        s, o = job
        cmd = [NVCC, *FLAGS, "-c", s, "-o", o] + (["-Xptxas", "-v"] if verbose else [])
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {s}:\n{r.stdout}\n{r.stderr}")
        return r.stderr

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        logs = list(ex.map(cc, jobs))
    if verbose:
        print("\n".join(logs))
    objs = [os.path.join(OBJ, src[:-3] + ".o") for src in _sources()]
    if jobs or not os.path.exists(LIB):
        r = subprocess.run([NVCC, "-shared", "-cudart", "shared", "-o", LIB, *objs], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose="-v" in sys.argv))
