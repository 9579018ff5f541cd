"""Builds oracle/_ref/libnerfshop_ref_camera.so: the reference's OWN camera-path arithmetic, compiled for the CPU.

TEST INFRASTRUCTURE ONLY (tests/test_camera_path_cpu.py pins nerfshop_b200/camera_path.py to it). Nothing under nerfshop_b200/ may import
or link it.

Cut out of the reference's tree (ref_build.REF) by signature and brace matching (oracle/ref_build.cut; never copied into the repository;
the cut-outs are deleted after the compile) and #included by oracle/ref_camera_driver.cpp:
  include/neural-graphics-primitives/camera_path.h   struct CameraKeyframe (m(), from_m, the matrix constructor, * and +), struct CameraPath
                                                      (get_keyframe, eval_camera_path), the lerp / spline declarations
  src/camera_path.cu                                   lerp, spline
This is host code in the reference, so it is compiled as oracle/ref_slices_build.py compiles the slice writers: g++ with -ffp-contract=off,
not the -mfma CPU build of the kernels. The reference's Eigen is absent: oracle/ref_shim_camera/Eigen/Dense stands in for the part used.
CameraPath's JSON (to_json / from_json / load / save) needs nlohmann's initializer lists and streams, which the repository's json
stand-in does not have; it is not part of this library.
"""
from __future__ import annotations

import os
import shutil
import subprocess

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


def _deps():
    deps = [DRIVER, os.path.abspath(__file__), os.path.abspath(ref_build.__file__)]
    for root, _, files in os.walk(SHIM):
        deps += [os.path.join(root, f) for f in files]
    return deps


def build(force: bool = False):
    """Returns the library path, or None when the reference's sources are absent and no prebuilt library exists."""
    if not ref_build.available():
        return LIB if os.path.exists(LIB) else None
    if not force and os.path.exists(LIB) and all(os.path.getmtime(d) <= os.path.getmtime(LIB) for d in _deps()):
        return LIB
    gen = os.path.join(ref_build.OUT_DIR, "gen_camera")
    shutil.rmtree(gen, ignore_errors=True)
    os.makedirs(gen, exist_ok=True)
    for name, (rel, anchors) in EXTRACTS.items():
        path = os.path.join(ref_build.REF, rel)
        with open(path, "r", encoding="utf-8", errors="replace") as fh:
            lines = fh.read().split("\n")
        parts = []
        for kind, anchor in anchors:
            a, b = ref_build.cut(lines, kind, anchor)
            parts.append(f"#line {a + 1} \"{path}\"\n" + "\n".join(lines[a:b + 1]) + "\n")
        with open(os.path.join(gen, name + ".inc"), "w") as fh:
            fh.write("\n".join(parts))
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    cmd = [cxx, "-std=c++17", "-O2", "-fPIC", "-shared", "-ffp-contract=off", "-fno-fast-math", "-w", "-I", SHIM, "-I", gen, DRIVER, "-o", LIB]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if os.environ.get("NSB_REF_KEEP_GEN") != "1":
        shutil.rmtree(gen, ignore_errors=True)
    if res.returncode != 0:
        raise RuntimeError("oracle/_ref camera build failed:\n" + res.stdout + res.stderr[-6000:])
    return LIB


if __name__ == "__main__":
    print(build(force=True))
