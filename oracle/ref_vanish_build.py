"""Builds oracle/_ref/libnerfshop_ref_vanish.so: libnerfshop_ref.so's sources plus the reference's OWN TetMesh::vanish, compiled for the CPU.

TEST INFRASTRUCTURE ONLY (tests/test_vanish_cpu.py pins the host restatement of vanish, which nsb_cage_vanish is tested against, to it).
Nothing under nerfshop_b200/ may import or link it.

Cut out of the reference's tree (ref_build.REF, NSB_REFERENCE_ROOT) by signature and brace matching (oracle/ref_build.cut; never
copied into the repository; the cut-outs are deleted after the compile) and #included by oracle/ref_vanish_driver.cpp after the whole
of oracle/ref_driver.cpp:
  src/editing/datastructures/tet_mesh.cu   the clear_cells static, clear_grid, TetMesh::vanish
The rest (every EXTRACTS entry of ref_build.py, the stand-ins of oracle/ref_shim/, the flags) is ref_build.build's. clear_grid runs
through the stand-in tcnn::linear_kernel, an OpenMP loop over the launch's threads.
"""
from __future__ import annotations

import os
import shutil
import subprocess

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


def _deps():
    deps = [DRIVER, ref_build.DRIVER, ref_build.COMMON, os.path.abspath(__file__), os.path.abspath(ref_build.__file__),
            os.path.join(HERE, "..", "include", "nerfshop_b200.h")]
    for root, _, files in os.walk(ref_build.SHIM):
        deps += [os.path.join(root, f) for f in files]
    return deps


def build(force: bool = False):
    """Returns the library path, or None when the reference's sources are absent and no prebuilt library exists."""
    if not ref_build.available():
        return LIB if os.path.exists(LIB) else None
    if not force and os.path.exists(LIB) and all(os.path.getmtime(d) <= os.path.getmtime(LIB) for d in _deps()):
        return LIB
    gen = os.path.join(ref_build.OUT_DIR, "gen_vanish")
    shutil.rmtree(gen, ignore_errors=True)
    ref_build.extract_all(gen)
    for name, (rel, items) in EXTRACTS.items():
        path = os.path.join(ref_build.REF, rel)
        with open(path, "r", encoding="utf-8", errors="replace") as fh:
            lines = fh.read().split("\n")
        parts = []
        for kind, pattern in items:
            a, b = ref_build.cut(lines, kind, pattern)
            parts.append(f"#line {a + 1} \"{path}\"\n" + "\n".join(lines[a:b + 1]) + "\n")
        with open(os.path.join(gen, name + ".inc"), "w") as fh:
            fh.write("\n".join(parts))
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    cmd = [cxx, "-std=c++17", "-O2", "-fPIC", "-shared", "-fopenmp", "-ffp-contract=fast", "-mfma", "-fno-fast-math",
           "-Wno-deprecated-declarations", "-Wno-attributes", "-w",
           "-I", ref_build.SHIM, "-I", gen, "-I", HERE, "-I", os.path.join(ref_build.REF, "include"), "-I", os.path.join(ref_build.REF, "src"),
           "-x", "c++", DRIVER, "-o", LIB]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if os.environ.get("NSB_REF_KEEP_GEN") != "1":
        shutil.rmtree(gen, ignore_errors=True)  # the cut-outs are reference source: they do not stay on disk
    if res.returncode != 0:
        raise RuntimeError("oracle/_ref vanish build failed:\n" + res.stdout + res.stderr[-6000:])
    return LIB


if __name__ == "__main__":
    print(build(force=True))
