"""Builds oracle/_ref/libnerfshop_ref_slices_cuda.so: the reference's OWN slice-export sources, compiled by nvcc for sm_90a (kernels) and
by its host compiler (the PNG writers).

TEST INFRASTRUCTURE ONLY (tests/test_gpu_slices.py pins nsb_rgba_on_grid, nsb_density_png, nsb_rgba_png and nerfshop_b200/slices.py to
it). Nothing under nerfshop_b200/ may import or link it.

Cut out of /root/reference by signature and brace matching (oracle/ref_build.cut; never copied into the repository; the cut-outs are
deleted after the compile) and #included by oracle/ref_slices_driver_cuda.cu:
  src/testbed_nerf.cu     generate_grid_samples_nerf_uniform_dir, compute_nerf_density
  src/marching_cubes.cu   save_density_grid_to_png, save_rgba_grid_to_png_sequence
The writers are host code: nvcc hands them to g++, which does not contract a * b + c without -mfma (-ffp-contract=off makes it explicit),
as the reference's host build computes their pixels. The reference's network (tiny-cuda-nn, absent) is not part of it: the tests run this
repository's nsb_inference between the kernels, its fp16 rows 0-3 cast to float standing in for Network::inference's float output (a
tiny-cuda-nn assumption: that inference writes the fp16 inference_mixed_precision output converted to float). Stand-ins for the absent
submodules: oracle/ref_shim_slices/ (stbi_write_png and tinylogger that record, and the out-of-line members of the reference's own
ThreadPool), then oracle/ref_shim/.
"""
from __future__ import annotations

import os
import shutil
import subprocess

from . import ref_build

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(ref_build.OUT_DIR, "libnerfshop_ref_slices_cuda.so")
DRIVER = os.path.join(HERE, "ref_slices_driver_cuda.cu")
SHIM = os.path.join(HERE, "ref_shim_slices")

EXTRACTS = {
    "marching_cubes_slices": ("src/marching_cubes.cu", [
        r"^void save_density_grid_to_png\(",
        r"^void save_rgba_grid_to_png_sequence\(",
    ]),
    "testbed_nerf_slices": ("src/testbed_nerf.cu", [
        r"^__global__ void generate_grid_samples_nerf_uniform_dir\(",
        r"^__global__ void compute_nerf_density\(",
    ]),
}


def _deps():
    deps = [DRIVER, os.path.abspath(__file__)]
    for d in (SHIM, ref_build.SHIM):
        for root, _, files in os.walk(d):
            deps += [os.path.join(root, f) for f in files]
    return deps


def build(force: bool = False):
    """Returns the library path, or None when the reference's sources are absent and no prebuilt library exists."""
    if not ref_build.available():
        return LIB if os.path.exists(LIB) else None
    if not force and os.path.exists(LIB) and all(os.path.getmtime(d) <= os.path.getmtime(LIB) for d in _deps()):
        return LIB
    gen = os.path.join(ref_build.OUT_DIR, "gen_slices")
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
           "-Xcompiler", "-fPIC", "-Xcompiler", "-ffp-contract=off", "-shared", "-w"] + (
           ["-ccbin", "/usr/bin/g++"] if os.path.exists("/usr/bin/g++") else []) + [
           "-I", SHIM, "-I", ref_build.SHIM, "-I", gen, "-I", os.path.join(ref_build.REF, "include"), "-I", os.path.join(ref_build.REF, "src"),
           DRIVER, "-o", LIB]
    if os.environ.get("NSB_REF_KEEP_GEN") == "1":
        cmd += ["--keep", "--keep-dir", gen]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if os.environ.get("NSB_REF_KEEP_GEN") != "1":
        shutil.rmtree(gen, ignore_errors=True)
    if res.returncode != 0:
        raise RuntimeError("oracle/_ref slices build failed:\n" + res.stdout + res.stderr[-6000:])
    return LIB


if __name__ == "__main__":
    print(build(force=True))
