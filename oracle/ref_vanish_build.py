"""Builds oracle/_ref/libnerfshop_ref_vanish.so: libnerfshop_ref.so's sources plus the reference's OWN TetMesh::vanish, compiled for the CPU.

TEST INFRASTRUCTURE ONLY (tests/test_vanish_cpu.py pins the host restatement of vanish, which nsb_cage_vanish is tested against, to it).
Nothing under nerfshop_b200/ may import or link it.

Cut out of the reference's tree (ref_build.REF, NSB_REFERENCE_ROOT) by signature and brace matching (oracle/ref_build.cut; never
copied into the repository; the cut-outs are deleted after the compile) and #included by oracle/ref_vanish_driver.cpp after the whole
of oracle/ref_driver.cpp:
  src/editing/datastructures/tet_mesh.cu   the clear_cells static, clear_grid, TetMesh::vanish
The rest (every EXTRACTS entry of ref_build.py, the stand-ins of oracle/ref_shim/, the flags ref_build.GXX_KERNELS) is ref_build.build's.
clear_grid runs through the stand-in tcnn::linear_kernel, an OpenMP loop over the launch's threads.
"""
from __future__ import annotations

import os

from . import ref_build

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(ref_build.OUT_DIR, "libnerfshop_ref_vanish.so")
DRIVER = os.path.join(HERE, "ref_vanish_driver.cpp")

EXTRACTS = {
    "tet_mesh_vanish": ("src/editing/datastructures/tet_mesh.cu", [
        ("stmt", r"^static std::vector<std::vector<int2>> clear_cells;"),
        ("fn", r"^__global__ void clear_grid\("),
        ("fn", r"^void TetMesh<float_t, point_t>::vanish\("),
    ]),
}


def build(force: bool = False):
    """Returns the library path, or None when the reference's sources are absent and no prebuilt library exists."""
    return ref_build.build_library(
        LIB, DRIVER, "gen_vanish",
        lambda gen: ref_build.GXX_KERNELS + ["-I", ref_build.SHIM, "-I", gen, "-I", HERE, *ref_build.REF_INCLUDES, "-x", "c++", DRIVER, "-o", LIB],
        lambda gen: ref_build.extract_all(gen) + ref_build.write_cutouts(EXTRACTS, gen), [ref_build.SHIM], __file__, force)


if __name__ == "__main__":
    print(build(force=True))
