"""Builds oracle/_ref/libnerfshop_ref_mesh_opt_cuda.so: the reference's OWN mesh optimisation gradient, compiled by nvcc for sm_90a.

TEST INFRASTRUCTURE ONLY (tests/test_gpu_mesh_optimise_ref.py pins nsb_mesh_optimise to it). Nothing under nerfshop_b200/ may import or link it.

Cut out of /root/reference by signature and brace matching (oracle/ref_build.cut; never copied into the repository; the cut-outs are deleted
after the compile) and #included by oracle/ref_mesh_opt_driver_cuda.cu:
  src/marching_cubes.cu   accumulate_1ring, compute_mesh_1ring, compute_mesh_opt_gradients_kernel, compute_mesh_opt_gradients
The reference's network and optimiser (tiny-cuda-nn, absent) are not part of it: the test runs nsb_density_gradient before it and the
restated Adam (oracle/mesh_opt_oracle.cpp) after it. Stand-ins for the absent submodules: oracle/ref_shim/. Flags are ref_mesh_build's.
"""
from __future__ import annotations

import os
import shutil
import subprocess

from . import ref_build

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(ref_build.OUT_DIR, "libnerfshop_ref_mesh_opt_cuda.so")
DRIVER = os.path.join(HERE, "ref_mesh_opt_driver_cuda.cu")

EXTRACTS = {
    "marching_cubes_opt": ("src/marching_cubes.cu", [
        r"^__global__ void accumulate_1ring\(",
        r"^void compute_mesh_1ring\(",
        r"^__global__ void compute_mesh_opt_gradients_kernel\(",
        r"^void compute_mesh_opt_gradients\(",
    ]),
}


def _deps():
    deps = [DRIVER, os.path.abspath(__file__)]
    for root, _, files in os.walk(ref_build.SHIM):
        deps += [os.path.join(root, f) for f in files]
    return deps


def build(force: bool = False):
    """Returns the library path, or None when /root/reference is absent and no prebuilt library exists."""
    if not ref_build.available():
        return LIB if os.path.exists(LIB) else None
    if not force and os.path.exists(LIB) and all(os.path.getmtime(d) <= os.path.getmtime(LIB) for d in _deps()):
        return LIB
    gen = os.path.join(ref_build.OUT_DIR, "gen_mesh_opt")
    shutil.rmtree(gen, ignore_errors=True)
    os.makedirs(gen, exist_ok=True)
    for name, (rel, anchors) in EXTRACTS.items():
        with open(os.path.join(ref_build.REF, rel), "r", encoding="utf-8", errors="replace") as fh:
            lines = fh.read().split("\n")
        parts = []
        for anchor in anchors:
            a, b = ref_build.cut(lines, "fn", anchor)
            parts.append(f"#line {a + 1} \"{os.path.join(ref_build.REF, rel)}\"\n" + "\n".join(lines[a:b + 1]) + "\n")
        with open(os.path.join(gen, name + ".inc"), "w") as fh:
            fh.write("\n".join(parts))
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--extended-lambda", "--expt-relaxed-constexpr",
           "-Xcompiler", "-fPIC", "-shared", "-w"] + (["-ccbin", "/usr/bin/g++"] if os.path.exists("/usr/bin/g++") else []) + [
           "-I", ref_build.SHIM, "-I", gen, "-I", os.path.join(ref_build.REF, "include"), "-I", os.path.join(ref_build.REF, "src"),
           DRIVER, "-o", LIB]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if os.environ.get("NSB_REF_KEEP_GEN") != "1":
        shutil.rmtree(gen, ignore_errors=True)
    if res.returncode != 0:
        raise RuntimeError("oracle/_ref mesh optimisation build failed:\n" + res.stdout + res.stderr[-6000:])
    return LIB


if __name__ == "__main__":
    print(build(force=True))
