"""Builds oracle/_ref/libnerfshop_ref_slices_cuda.so: the reference's OWN slice-export sources, compiled by nvcc for sm_90a (kernels) and
by its host compiler (the PNG writers).

TEST INFRASTRUCTURE ONLY (tests/test_gpu_slices.py pins nsb_rgba_on_grid, nsb_density_png, nsb_rgba_png and nerfshop_b200/slices.py to
it). Nothing under nerfshop_b200/ may import or link it.

Cut out of /root/reference by signature and brace matching (oracle/ref_build.cut; never copied into the repository; the cut-outs are
deleted after the compile) and #included by oracle/ref_slices_driver_cuda.cu:
  src/testbed_nerf.cu     generate_grid_samples_nerf_uniform_dir, compute_nerf_density
  src/marching_cubes.cu   save_density_grid_to_png, save_rgba_grid_to_png_sequence
The writers are host code: nvcc hands them to g++, which does not contract a * b + c without -mfma (-ffp-contract=off makes it explicit),
as the reference's host build computes their pixels: the flags are ref_build.NVCC plus -Xcompiler -ffp-contract=off. The reference's
network (tiny-cuda-nn, absent) is not part of it: the tests run this repository's nsb_inference between the kernels, its fp16 rows 0-3
cast to float standing in for Network::inference's float output (a tiny-cuda-nn assumption: that inference writes the fp16
inference_mixed_precision output converted to float). Stand-ins for the absent submodules: oracle/ref_shim_slices/ (stbi_write_png and
tinylogger that record, and the out-of-line members of the reference's own ThreadPool), then oracle/ref_shim/.
"""
from __future__ import annotations

import os

from . import ref_build

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(ref_build.OUT_DIR, "libnerfshop_ref_slices_cuda.so")
DRIVER = os.path.join(HERE, "ref_slices_driver_cuda.cu")
SHIM = os.path.join(HERE, "ref_shim_slices")

EXTRACTS = {
    "marching_cubes_slices": ("src/marching_cubes.cu", [
        ("fn", r"^void save_density_grid_to_png\("),
        ("fn", r"^void save_rgba_grid_to_png_sequence\("),
    ]),
    "testbed_nerf_slices": ("src/testbed_nerf.cu", [
        ("fn", r"^__global__ void generate_grid_samples_nerf_uniform_dir\("),
        ("fn", r"^__global__ void compute_nerf_density\("),
    ]),
}


def build(force: bool = False):
    """Returns the library path, or None when the reference's sources are absent and no prebuilt library exists."""
    return ref_build.build_library(
        LIB, DRIVER, "gen_slices",
        lambda gen: ref_build.NVCC + ["-Xcompiler", "-ffp-contract=off",
                                      "-I", SHIM, "-I", ref_build.SHIM, "-I", gen, *ref_build.REF_INCLUDES, DRIVER, "-o", LIB],
        lambda gen: ref_build.write_cutouts(EXTRACTS, gen), [SHIM, ref_build.SHIM], __file__, force)


if __name__ == "__main__":
    print(build(force=True))
