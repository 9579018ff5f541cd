"""Builds oracle/_ref/libnerfshop_ref_video_cuda.so: the reference's render_frame sequence per sub-frame of Testbed::render_to_cpu
(clear_frame, render_nerf, accumulate_kernel, tonemap_kernel), compiled by nvcc for sm_90a.

TEST INFRASTRUCTURE ONLY (tests/test_gpu_camera_path.py pins nsb_render_accumulate to it). Nothing under nerfshop_b200/ may import or
link it.

oracle/ref_video_driver_cuda.cu includes the whole of oracle/ref_driver_cuda.cu, so the reference sources are those of
ref_build.build_cuda (ref_build.EXTRACTS, cut out by signature, deleted after the compile; accumulate_kernel and tonemap_kernel among
them), with the same stand-ins and flags (ref_build.NVCC plus -lineinfo). The network is the caller's nsb_inference, as for
libnerfshop_ref_cuda.so.
"""
from __future__ import annotations

import os

from . import ref_build

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(ref_build.OUT_DIR, "libnerfshop_ref_video_cuda.so")
DRIVER = os.path.join(HERE, "ref_video_driver_cuda.cu")


def build(force: bool = False):
    """Returns the library path, or None when the reference's sources are absent and no prebuilt library exists."""
    return ref_build.build_library(
        LIB, DRIVER, "gen_video",
        lambda gen: ref_build.NVCC + ["-lineinfo", "-I", HERE, "-I", ref_build.SHIM, "-I", gen, *ref_build.REF_INCLUDES, DRIVER, "-o", LIB],
        ref_build.extract_all, [ref_build.SHIM], __file__, force)


if __name__ == "__main__":
    print(build(force=True))
