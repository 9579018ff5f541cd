"""Builds oracle/_ref/libnerfshop_ref_camera.so: the reference's OWN camera-path arithmetic, compiled for the CPU.

TEST INFRASTRUCTURE ONLY (tests/test_camera_path_cpu.py pins nerfshop_b200/camera_path.py to it). Nothing under nerfshop_b200/ may import
or link it.

Cut out of the reference's tree (ref_build.REF) by signature and brace matching (oracle/ref_build.cut; never copied into the repository;
the cut-outs are deleted after the compile) and #included by oracle/ref_camera_driver.cpp:
  include/neural-graphics-primitives/camera_path.h   struct CameraKeyframe (m(), from_m, the matrix constructor, * and +), struct CameraPath
                                                      (get_keyframe, eval_camera_path), the lerp / spline declarations
  src/camera_path.cu                                   lerp, spline
This is host code in the reference, so it is compiled as oracle/ref_slices_build.py compiles the slice writers: g++ with -ffp-contract=off
(ref_build.GXX_HOST), not the -mfma CPU build of the kernels. The reference's Eigen is absent: oracle/ref_shim_camera/Eigen/Dense stands in
for the part used.
CameraPath's JSON (to_json / from_json / load / save) needs nlohmann's initializer lists and streams, which the repository's json
stand-in does not have; it is not part of this library.
"""
from __future__ import annotations

import os

from . import ref_build

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(ref_build.OUT_DIR, "libnerfshop_ref_camera.so")
DRIVER = os.path.join(HERE, "ref_camera_driver.cpp")
SHIM = os.path.join(HERE, "ref_shim_camera")

EXTRACTS = {
    "camera_path_h": ("include/neural-graphics-primitives/camera_path.h", [
        ("fn", r"^struct CameraKeyframe \{"),
        ("stmt", r"^CameraKeyframe lerp\("),
        ("stmt", r"^CameraKeyframe spline\("),
        ("fn", r"^struct CameraPath \{"),
    ]),
    "camera_path_cu": ("src/camera_path.cu", [("fn", r"^CameraKeyframe lerp\("), ("fn", r"^CameraKeyframe spline\(")]),
}


def build(force: bool = False):
    """Returns the library path, or None when the reference's sources are absent and no prebuilt library exists."""
    return ref_build.build_library(
        LIB, DRIVER, "gen_camera",
        lambda gen: ref_build.GXX_HOST + ["-I", SHIM, "-I", gen, DRIVER, "-o", LIB],
        lambda gen: ref_build.write_cutouts(EXTRACTS, gen), [SHIM], __file__, force)


if __name__ == "__main__":
    print(build(force=True))
