"""Builds oracle/_ref/libnerfshop_ref_mesh_cuda.so: the reference's OWN mesh-extraction sources, compiled by nvcc for sm_90a.

TEST INFRASTRUCTURE ONLY (tests/test_gpu_mesh_ref.py pins nsb_density_on_grid, nsb_marching_cubes, nsb_mesh_shade and
nerfshop_b200/mesh.py to it). Nothing under nerfshop_b200/ may import or link it.

Cut out of /root/reference by signature and brace matching (oracle/ref_build.cut; never copied into the repository; the cut-outs
are deleted after the compile) and #included by oracle/ref_mesh_driver_cuda.cu:
  src/marching_cubes.cu   get_marching_cubes_res, gen_vertices, accumulate_1ring, gen_faces, compute_mesh_1ring, marching_cubes_gpu, save_mesh
  src/testbed_nerf.cu     generate_grid_samples_nerf_uniform, grid_samples_half_to_float, generate_nerf_network_inputs_from_positions,
                          extract_srgb_with_activation
The reference's network (tiny-cuda-nn, absent) is not part of it: the tests run this repository's nsb_density / nsb_inference between
the reference's kernels, as the render-path parity does. Stand-ins for the absent submodules: oracle/ref_shim/ and oracle/ref_shim_mesh/
(filesystem/path.h, stb_image_write.h). Flags: ref_build.NVCC.
"""
from __future__ import annotations

import os

from . import ref_build

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(ref_build.OUT_DIR, "libnerfshop_ref_mesh_cuda.so")
DRIVER = os.path.join(HERE, "ref_mesh_driver_cuda.cu")
SHIM = os.path.join(HERE, "ref_shim_mesh")

EXTRACTS = {
    "marching_cubes_mesh": ("src/marching_cubes.cu", [
        ("fn", r"^Vector3i get_marching_cubes_res\("),
        ("fn", r"^__global__ void gen_vertices\("),
        ("fn", r"^__global__ void accumulate_1ring\("),
        ("fn", r"^__global__ void gen_faces\("),
        ("fn", r"^void compute_mesh_1ring\("),
        ("fn", r"^void marching_cubes_gpu\("),
        ("fn", r"^void save_mesh\("),
    ]),
    "testbed_nerf_mesh": ("src/testbed_nerf.cu", [
        ("fn", r"^__global__ void generate_grid_samples_nerf_uniform\("),
        ("fn", r"^__global__ void grid_samples_half_to_float\("),
        ("fn", r"^__global__ void generate_nerf_network_inputs_from_positions\("),
        ("fn", r"^__global__ void extract_srgb_with_activation\("),
    ]),
}


def build(force: bool = False):
    """Returns the library path, or None when /root/reference is absent and no prebuilt library exists."""
    return ref_build.build_library(
        LIB, DRIVER, "gen_mesh",
        lambda gen: ref_build.NVCC + ["-I", SHIM, "-I", ref_build.SHIM, "-I", gen, *ref_build.REF_INCLUDES, DRIVER, "-o", LIB],
        lambda gen: ref_build.write_cutouts(EXTRACTS, gen), [SHIM, ref_build.SHIM], __file__, force)


if __name__ == "__main__":
    print(build(force=True))
