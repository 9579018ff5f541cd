"""Builds nerfshop_b200/lib/libnerfshop_b200.so (hand-written sm_90a CUDA + host C++), in-tree.

nvcc cross-compiles without a GPU; the .so is git-ignored but travels to the GPU box with the repo snapshot.
"""
from __future__ import annotations

import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_DIR = os.path.join(_HERE, "lib")
LIB = os.path.join(LIB_DIR, "libnerfshop_b200.so")
SOURCES = ["nsb_kernels.cu", "nsb_host_geometry.cpp"]
HEADERS = sorted(f for f in os.listdir(CSRC) if f.endswith((".cuh", ".h", ".hpp"))) + [
    os.path.join("..", "..", "include", "nerfshop_b200.h"), os.path.join("..", "host", "nerfshop_host.hpp")]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fno-fast-math", "-shared",
]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build_variant(name: str, defines) -> str:
    """An experiment build next to the product library: lib/libnerfshop_b200_<name>.so with extra -D flags (tools/ only)."""
    out = os.path.join(LIB_DIR, f"libnerfshop_b200_{name}.so")
    os.makedirs(LIB_DIR, exist_ok=True)
    ccbin = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else None
    cmd = [_nvcc()] + NVCC_FLAGS + (["-ccbin", ccbin] if ccbin else []) + [f"-D{d}" for d in defines] + ["-o", out] + [os.path.join(CSRC, s) for s in SOURCES]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    return out


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    os.makedirs(LIB_DIR, exist_ok=True)
    env = dict(os.environ)
    # the image exports CXX=/opt/gcc/bin/g++ (a wrapper); let nvcc pick the distro host compiler
    ccbin = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else None
    cmd = [_nvcc()] + NVCC_FLAGS + (["-ccbin", ccbin] if ccbin else []) + (["-Xptxas", "-v"] if verbose else [])
    cmd += ["-o", LIB] + [os.path.join(CSRC, s) for s in SOURCES]
    res = subprocess.run(cmd, capture_output=True, text=True, env=env)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    if verbose:
        print(res.stderr)
    return LIB


if __name__ == "__main__":
    import sys

    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
