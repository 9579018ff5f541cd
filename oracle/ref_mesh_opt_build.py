"""Builds oracle/_ref/libnerfshop_ref_mesh_opt_cuda.so: the reference's OWN mesh optimisation gradient, compiled by nvcc for sm_90a.

TEST INFRASTRUCTURE ONLY (tests/test_gpu_mesh_optimise_ref.py pins nsb_mesh_optimise to it). Nothing under nerfshop_b200/ may import or link it.

Cut out of /root/reference by signature and brace matching (oracle/ref_build.cut; never copied into the repository; the cut-outs are deleted
after the compile) and #included by oracle/ref_mesh_opt_driver_cuda.cu:
  src/marching_cubes.cu   accumulate_1ring, compute_mesh_1ring, compute_mesh_opt_gradients_kernel, compute_mesh_opt_gradients
The reference's network and optimiser (tiny-cuda-nn, absent) are not part of it: the test runs nsb_density_gradient before it and the
restated Adam (oracle/mesh_opt_oracle.cpp) after it. Stand-ins for the absent submodules: oracle/ref_shim/. Flags: ref_build.NVCC.
"""
from __future__ import annotations

import os

from . import ref_build

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(ref_build.OUT_DIR, "libnerfshop_ref_mesh_opt_cuda.so")
DRIVER = os.path.join(HERE, "ref_mesh_opt_driver_cuda.cu")

EXTRACTS = {
    "marching_cubes_opt": ("src/marching_cubes.cu", [
        ("fn", r"^__global__ void accumulate_1ring\("),
        ("fn", r"^void compute_mesh_1ring\("),
        ("fn", r"^__global__ void compute_mesh_opt_gradients_kernel\("),
        ("fn", r"^void compute_mesh_opt_gradients\("),
    ]),
}


def build(force: bool = False):
    """Returns the library path, or None when /root/reference is absent and no prebuilt library exists."""
    return ref_build.build_library(
        LIB, DRIVER, "gen_mesh_opt",
        lambda gen: ref_build.NVCC + ["-I", ref_build.SHIM, "-I", gen, *ref_build.REF_INCLUDES, DRIVER, "-o", LIB],
        lambda gen: ref_build.write_cutouts(EXTRACTS, gen), [ref_build.SHIM], __file__, force)


if __name__ == "__main__":
    print(build(force=True))
