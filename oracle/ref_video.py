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
        if hasattr(l, "refvid_postprocess"):  # a prebuilt library from before the entry point lacks it (serves_postprocess)
            l.refvid_postprocess.argtypes = [V, C.c_int, C.c_uint32, C.c_int, C.c_int, C.c_int, V, V, C.POINTER(C.c_float), C.c_int, V]
        _lib = l
    return _lib


def serves_postprocess() -> bool:
    """The library exists and has refvid_postprocess. A prebuilt one older than that entry point does not: the tests then replay the
    reference's stored results, as tests/ref_golden.py does for oracle/ref.py's later entry points."""
    return ref_video_build.build() is not None and hasattr(lib(), "refvid_postprocess")


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


def tonemap_rows(tms) -> np.ndarray:
    """NsbTonemaps -> the [n, 9] float32 rows refvid_postprocess reads (colour space aside, which the accumulation fixes)."""
    return np.array([[t.exposure, *t.background_color, t.output_color_space, t.tonemap_curve, t.clamp_output_color, 0.0] for t in tms], np.float32)


def postprocess(frames, spp0: int, color_space: int, acc0=None, tm_rows=None):
    """The reference's accumulate_kernel and tonemap_kernel on caller buffers, launched as CudaRenderBuffer does (16x8 blocks).

    frames: float32 [n, H, W, 4] accumulated in order with sample counts spp0, spp0 + 1, ... (the accumulation is zeroed when the count is
    0, else it starts from acc0 [H, W, 4]); n may be 0 to tonemap acc0 itself. tm_rows: tonemap_rows(...) or None.
    Returns (the accumulation after every call [H*W, n, 4], every tonemapped surface [H*W, n_tm, 4] or None): pixel-major, so a stored
    row sample keeps whole pixels."""
    import torch

    l = lib()
    frames = np.ascontiguousarray(frames, np.float32)
    n, H, W = frames.shape[0], frames.shape[1], frames.shape[2]
    if acc0 is not None:
        H, W = acc0.shape[0], acc0.shape[1]
    px = H * W
    f_dev = torch.from_numpy(frames).cuda() if n else None
    acc = torch.from_numpy(np.ascontiguousarray(acc0, np.float32)).cuda() if acc0 is not None else torch.zeros((H, W, 4), dtype=torch.float32, device="cuda")
    hist = torch.empty((max(n, 1), px, 4), dtype=torch.float32, device="cuda")
    rows = None if tm_rows is None else np.ascontiguousarray(tm_rows, np.float32)
    n_tm = 0 if rows is None else rows.shape[0]
    out = torch.empty((max(n_tm, 1), px, 4), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    rc = l.refvid_postprocess(f_dev.data_ptr() if n else None, n, spp0, W, H, color_space, acc.data_ptr(), hist.data_ptr() if n else None,
                              rows.ctypes.data_as(C.POINTER(C.c_float)) if n_tm else None, n_tm, out.data_ptr() if n_tm else None)
    assert rc == 0
    hist = hist[:n].permute(1, 0, 2).contiguous().cpu().numpy() if n else None
    return hist, (out.permute(1, 0, 2).contiguous().cpu().numpy() if n_tm else None)
