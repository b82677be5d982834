"""Build libmickey_b200.so (hand-written CUDA for sm_90a) in-tree with nvcc.

    python -m mickey_b200.build            # incremental
    python -m mickey_b200.build --force

The library is placed at mickey_b200/_C/libmickey_b200.so (git-ignored).  There is deliberately no CPU build and no other architecture.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT_DIR = os.path.join(HERE, "_C")
LIB = os.path.join(OUT_DIR, "libmickey_b200.so")
SOURCES = ["gemm.cu", "vit_ops.cu", "attention_tc.cu", "head_ops.cu", "ransac.cu", "io_ops.cu", "matches.cu", "loss.cu", "loss_tail.cu", "matcher_grad.cu", "head_transformer.cu",
           "resblock.cu", "head_out.cu", "mapfree_eval.cu", "engine.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _deps():
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    hdrs.append(os.path.join(os.path.dirname(HERE), "include", "mickey_b200.h"))
    return hdrs


def _stale(target, srcs):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in srcs)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OUT_DIR, exist_ok=True)
    hdrs = _deps()
    objs, jobs = [], []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(OUT_DIR, src.replace(".cu", ".o"))
        objs.append(o)
        if force or _stale(o, [s] + hdrs):
            jobs.append([NVCC, *FLAGS, "-c", s, "-o", o])

    def run(cmd):
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed:\n{' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
        return r

    with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 1) or 1) as ex:
        list(ex.map(run, jobs))
    if jobs or force or _stale(LIB, objs):
        run([NVCC, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a"])
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose=True)
    print("built", path)
