"""Build libkvb.so (sm_90a) in-tree with nvcc.  No torch involved: the library is plain CUDA runtime + C ABI.

    python llm-d-kv-cache_b200/build.py [--force] [--verbose]
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libkvb.so")
OBJ = os.path.join(HERE, "build")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC,-O3,-Wall,-Wno-unused-function",
    "-I", os.path.join(ROOT, "include"), "-I", CSRC,
]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found (needed to build libkvb.so for sm_90a)")


def sources() -> list[str]:
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cu", ".cpp")))


def _stale(target: str, deps: list[str]) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    srcs = sources()
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    headers.append(os.path.join(ROOT, "include", "kvb.h"))
    headers.append(os.path.abspath(__file__))
    if not force and not _stale(LIB, srcs + headers):
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    nvcc = _nvcc()
    objs, procs = [], []
    for s in srcs:
        o = os.path.join(OBJ, os.path.basename(s) + ".o")
        objs.append(o)
        if force or _stale(o, [s] + headers):
            cmd = [nvcc, *NVCC_FLAGS, "-x", "cu", "-c", s, "-o", o]
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
                print(" ".join(cmd), flush=True)
            procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for s, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            print(f"--- {os.path.basename(s)}\n{out}", flush=True)
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed building libkvb.so")
    cmd = [nvcc, "-shared", "-o", LIB + ".tmp", *objs, "-gencode", "arch=compute_90a,code=sm_90a",
           "-Xcompiler", "-fPIC", "-lpthread", "-ldl", "-lrt",
           "-Xlinker", "--no-undefined"]  # a missing definition must fail the build, not the first dlopen on a GPU host
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        print(r.stdout)
        raise RuntimeError("link failed for libkvb.so")
    os.replace(LIB + ".tmp", LIB)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
