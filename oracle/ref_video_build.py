"""Builds oracle/_ref/libnerfshop_ref_video_cuda.so: the reference's render_frame sequence per sub-frame of Testbed::render_to_cpu
(clear_frame, render_nerf, accumulate_kernel, tonemap_kernel), compiled by nvcc for sm_90a.

TEST INFRASTRUCTURE ONLY (tests/test_gpu_camera_path.py pins nsb_render_accumulate to it). Nothing under nerfshop_b200/ may import or
link it.

oracle/ref_video_driver_cuda.cu includes the whole of oracle/ref_driver_cuda.cu, so the reference sources are those of
ref_build.build_cuda (ref_build.EXTRACTS, cut out by signature, deleted after the compile; accumulate_kernel and tonemap_kernel among
them), with the same stand-ins and flags. The network is the caller's nsb_inference, as for libnerfshop_ref_cuda.so.
"""
from __future__ import annotations

import os
import shutil
import subprocess

from . import ref_build

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(ref_build.OUT_DIR, "libnerfshop_ref_video_cuda.so")
DRIVER = os.path.join(HERE, "ref_video_driver_cuda.cu")


def _deps():
    deps = [DRIVER, ref_build.DRIVER_CUDA, ref_build.COMMON, os.path.abspath(__file__), os.path.abspath(ref_build.__file__),
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
    gen = os.path.join(ref_build.OUT_DIR, "gen_video")
    shutil.rmtree(gen, ignore_errors=True)
    ref_build.extract_all(gen)
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo", "--extended-lambda", "--expt-relaxed-constexpr",
           "-Xcompiler", "-fPIC", "-shared", "-w"] + (["-ccbin", "/usr/bin/g++"] if os.path.exists("/usr/bin/g++") else []) + [
           "-I", HERE, "-I", ref_build.SHIM, "-I", gen, "-I", os.path.join(ref_build.REF, "include"), "-I", os.path.join(ref_build.REF, "src"),
           DRIVER, "-o", LIB]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if os.environ.get("NSB_REF_KEEP_GEN") != "1":
        shutil.rmtree(gen, ignore_errors=True)
    if res.returncode != 0:
        raise RuntimeError("oracle/_ref video build failed:\n" + res.stdout + res.stderr[-6000:])
    return LIB


if __name__ == "__main__":
    print(build(force=True))
