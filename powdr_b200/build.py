"""Build the sm_90a shared library in-tree (powdr_b200/_lib/libpowdr_b200.so) with nvcc.

One CUDA translation unit (csrc/capi.cu) plus the host-only transcript permutation (csrc/transcript_host.cpp, g++) -> one .so
exporting the C ABI of include/powdr_b200.h.  Cross-compiles without a GPU.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "_lib")
LIB = os.path.join(LIB_DIR, "libpowdr_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CXX = os.environ.get("CXX", "/usr/bin/g++")
FLAGS = ["-std=c++17", "-O3", "-ldl", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
         "-Xcompiler", "-fPIC", "-shared", "-ccbin", "/usr/bin/g++"]


def sources():
    out = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC))]
    inc = os.path.join(os.path.dirname(HERE), "include")
    out += [os.path.join(inc, f) for f in sorted(os.listdir(inc))]
    return out


def stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(s) > t for s in sources())


def build(force=False, verbose=False):
    if not force and not stale():
        return LIB
    os.makedirs(LIB_DIR, exist_ok=True)
    host_obj = os.path.join(LIB_DIR, "transcript_host.o")
    subprocess.check_call([CXX, "-std=c++17", "-O3", "-fPIC", "-c", os.path.join(CSRC, "transcript_host.cpp"), "-o", host_obj])
    cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB, os.path.join(CSRC, "capi.cu"), host_obj]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
