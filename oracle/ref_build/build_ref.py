#!/usr/bin/env python
"""Build the UNMODIFIED reference offload engine into oracle/_ref/ (test infrastructure).

Compiles the reference's own sources *where they lie* under /root/reference
(kv_connectors/llmd_fs_backend/csrc/storage, source list = its setup.py:21-30) with
torch.utils.cpp_extension for sm_90a.  Nothing is copied into this repo; the only
addition is shim/numa.h (libnuma is absent from the image, see the header).
Output: oracle/_ref/storage_offload_ref.so  (git-ignored).

Used by bench.py --impl reference and bench.py's cpu_baseline leg as the reference arm.
"""
import os
import sys

REF = os.environ.get("KVB_REFERENCE_ROOT", "/root/reference")
CSRC = os.path.join(REF, "kv_connectors/llmd_fs_backend/csrc/storage")
HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(os.path.dirname(HERE), "_ref")
NAME = "storage_offload_ref"

SOURCES = [
    "storage_offload.cpp",
    "storage_offload_bindings.cpp",
    "numa_utils.cpp",
    "backends/fs_io/file_io.cpp",
    "thread_pool.cpp",
    "tensor_copier.cu",
    "tensor_copier_kernels.cu",
    "backends/fs_gds/gds_file_io.cpp",
]


def build(verbose: bool = False) -> str | None:
    so = os.path.join(OUT, NAME + ".so")
    if not os.path.isdir(CSRC):
        return so if os.path.exists(so) else None
    if os.path.exists(so):
        newest = max(os.path.getmtime(os.path.join(CSRC, s)) for s in SOURCES)
        if os.path.getmtime(so) >= newest:
            return so
    os.makedirs(OUT, exist_ok=True)
    # The image's default CXX (/opt/gcc/bin/g++ wrapper) links libstdc++ STATICALLY; a second libstdc++ inside a
    # torch extension segfaults at first iostream use (the reference's own setup.py:52-56 warns about this), so
    # build with the distribution compiler, which links libstdc++.so.6 dynamically.
    for var, exe in (("CXX", "/usr/bin/g++"), ("CC", "/usr/bin/gcc")):
        if os.path.exists(exe):
            os.environ[var] = exe
    os.environ.setdefault("TORCH_CUDA_ARCH_LIST", "9.0a")
    os.environ.setdefault("MAX_JOBS", "8")
    from torch.utils.cpp_extension import load

    load(
        name=NAME,
        sources=[os.path.join(CSRC, s) for s in SOURCES],
        extra_include_paths=[
            os.path.join(HERE, "shim"),
            CSRC,
            os.path.join(CSRC, "backends/fs_io"),
            os.path.join(CSRC, "backends/fs_gds"),
        ],
        extra_cflags=["-O3", "-std=c++17", "-fopenmp"],
        extra_cuda_cflags=["-O3", "-std=c++17", "-Xcompiler", "-fopenmp", "-ccbin", os.environ.get("CXX", "g++")],
        extra_ldflags=["-ldl"],
        build_directory=OUT,
        is_python_module=False,
        verbose=verbose,
    )
    return so if os.path.exists(so) else None


if __name__ == "__main__":
    p = build(verbose=True)
    print("reference engine:", p)
    sys.exit(0 if p else 1)
