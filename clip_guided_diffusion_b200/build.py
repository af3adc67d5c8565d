"""Build libcgd_b200.so in-tree with nvcc for sm_90a (H100; no torch extension machinery: the library is a plain
C-ABI shared object loaded with ctypes)."""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libcgd_b200.so")
SOURCES = ["api.cu", "conv_tc.cu", "conv_narrow.cu", "norm.cu", "norm_fused.cu", "norm_grid.cu", "norm_grid2.cu", "elementwise.cu", "attention.cu", "attention_small.cu", "attention_flash.cu", "guidance.cu", "augs.cu", "lpips.cu", "linear_small.cu", "resample.cu", "text.cu", "autograd.cu", "clip_autograd.cu", "losses.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
              "--use_fast_math=false"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    nvcc = _nvcc()
    flags = [f for f in NVCC_FLAGS if not f.startswith("--use_fast_math")] + os.environ.get("CGD_NVCC_EXTRA", "").split()  # e.g. -DCGD_SIGMOID_EX2RCP (A/B builds)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(HERE, "..", "include", "cgd_b200.h"))
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    jobs = []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(objdir, src.replace(".cu", ".o"))
        if force or _stale(o, [s] + headers):
            jobs.append((s, o))

    def cc(job):
        s, o = job
        cmd = [nvcc] + flags + ["-c", s, "-o", o]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {s}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print("compiled", os.path.basename(s), file=sys.stderr)

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        list(ex.map(cc, jobs))
    objs = [os.path.join(objdir, src.replace(".cu", ".o")) for src in SOURCES]
    if force or jobs or _stale(LIB, objs):
        cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB] + objs + ["-Xcompiler", "-fPIC", "-cudart", "static"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
