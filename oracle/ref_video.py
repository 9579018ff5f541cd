"""Python side of oracle/_ref/libnerfshop_ref_video_cuda.so (oracle/ref_video_build.py): the reference's render_frame sequence per
sub-frame of Testbed::render_to_cpu. TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C

import numpy as np

from nerfshop_b200 import abi

from . import ref_video_build

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        path = ref_video_build.build()
        if path is None:
            raise RuntimeError("oracle/_ref: no libnerfshop_ref_video_cuda.so (built where the reference's sources exist; it travels with the repo)")
        l = C.CDLL(path)
        V = C.c_void_p
        l.refcu_create.restype = V  # the whole of ref_driver_cuda.cu is in this library: its own scene
        l.refcu_create.argtypes = [V, C.POINTER(abi.NsbEditOp), C.c_int]
        l.refcu_destroy.argtypes = [V]
        l.refcu_destroy.restype = None
        l.refvid_render_to_cpu.argtypes = [V, C.POINTER(abi.NsbFrame), C.c_int, V, V, C.c_float, C.POINTER(C.c_float), C.c_int, C.c_int, C.c_int, C.c_int,
                                           V, V, V, V]
        _lib = l
    return _lib


def render_to_cpu(bitfield, ops, frames, renderer, tm: abi.NsbTonemap) -> np.ndarray:
    """The reference's clear_frame -> render_nerf -> accumulate_kernel -> tonemap_kernel for every sub-frame (frames: NsbFrames of one
    size, spp_index = the accumulate's sample count), the tonemapped surface after the last one as float32 [H, W, 4]. The network is
    `renderer`'s nsb_inference (tiny-cuda-nn is absent)."""
    import torch

    l = lib()
    from .ref import _ops_array

    b = np.ascontiguousarray(bitfield, np.uint8)
    arr, n_ops = _ops_array(ops)
    h = l.refcu_create(b.ctypes.data, arr, n_ops)
    assert h, "refcu_create failed"
    try:
        W, H = frames[0].width, frames[0].height
        fb = torch.zeros((H, W, 4), dtype=torch.float32, device="cuda")
        depth = torch.zeros((H, W), dtype=torch.float32, device="cuda")
        acc = torch.zeros_like(fb)
        out = torch.zeros_like(fb)
        fa = (abi.NsbFrame * len(frames))(*frames)
        bg = (C.c_float * 4)(*tm.background_color)
        fn = C.cast(renderer.lib.nsb_inference, C.c_void_p)
        torch.cuda.synchronize()
        rc = l.refvid_render_to_cpu(h, fa, len(frames), fn, renderer.ctx, tm.exposure, bg, tm.color_space, tm.output_color_space, tm.tonemap_curve,
                                    tm.clamp_output_color, fb.data_ptr(), depth.data_ptr(), acc.data_ptr(), out.data_ptr())
        assert rc == 0
        return out.cpu().numpy()
    finally:
        l.refcu_destroy(h)
