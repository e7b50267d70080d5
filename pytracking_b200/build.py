"""Builds pytracking_b200/libb200trk.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU)."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build", "sm_90a")      # objects of another target are never linked in
LIB = os.path.join(HERE, "libb200trk.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17",
                 "-Xcompiler", "-fPIC", "-Xcompiler", "-Wall", "-diag-suppress", "177",
                 "-Xcompiler", "-ffp-contract=off"]      # host float32 state arithmetic must not be fused (dimp_tracker.cu)


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _newest_header():
    t = os.path.getmtime(os.path.join(HERE, "..", "include", "b200trk.h"))
    for f in os.listdir(CSRC):
        if f.endswith((".cuh", ".h")):
            t = max(t, os.path.getmtime(os.path.join(CSRC, f)))
    return t


def build_library(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    hdr_t = _newest_header()
    jobs = []
    for src in _sources():
        s = os.path.join(CSRC, src)
        o = os.path.join(OBJ, src[:-3] + ".o")
        if force or not os.path.exists(o) or os.path.getmtime(o) < max(os.path.getmtime(s), hdr_t):
            jobs.append((s, o))

    def compile_one(job):
        s, o = job
        cmd = [NVCC] + FLAGS + ["-c", s, "-o", o]
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (s, r.stdout, r.stderr))
        return o

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(compile_one, jobs))
    objs = [os.path.join(OBJ, s[:-3] + ".o") for s in _sources()]
    if jobs or force or not os.path.exists(LIB):
        cmd = [NVCC, "-shared"] + ARCH + ["-o", LIB] + objs
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


if __name__ == "__main__":
    print(build_library(force="--force" in sys.argv, verbose=True))
