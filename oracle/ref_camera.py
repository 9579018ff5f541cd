"""Python side of oracle/_ref/libnerfshop_ref_camera.so (oracle/ref_camera_build.py): the reference's CameraKeyframe and
CameraPath::eval_camera_path. Keyframes are float32 rows of 11: R (x, y, z, w), T, slice, scale, fov, dof. TEST INFRASTRUCTURE ONLY."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import ref_camera_build

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        path = ref_camera_build.build()
        if path is None:
            raise RuntimeError("oracle/_ref: no libnerfshop_ref_camera.so (built where the reference's sources exist)")
        _lib = C.CDLL(path)
        V, F = C.c_void_p, C.c_float
        _lib.refcam_m.argtypes = [V, V]
        _lib.refcam_from_matrix.argtypes = [V, F, F, F, F, V]
        _lib.refcam_eval.argtypes = [V, C.c_int, V, C.c_int, V]
        for f in (_lib.refcam_m, _lib.refcam_from_matrix, _lib.refcam_eval):
            f.restype = None
    return _lib


def m(kfs) -> np.ndarray:
    """CameraKeyframe::m() of each row: [n, 12] column-major."""
    k = np.ascontiguousarray(kfs, np.float32).reshape(-1, 11)
    out = np.zeros((k.shape[0], 12), np.float32)
    for i in range(k.shape[0]):
        lib().refcam_m(k[i].ctypes.data, out[i].ctypes.data)
    return out


def from_matrix(mats) -> np.ndarray:
    """CameraKeyframe(Matrix<float, 3, 4>, 0, 1, 50, 0) of each column-major matrix [n, 12]: [n, 11]."""
    ms = np.ascontiguousarray(mats, np.float32).reshape(-1, 12)
    out = np.zeros((ms.shape[0], 11), np.float32)
    for i in range(ms.shape[0]):
        lib().refcam_from_matrix(ms[i].ctypes.data, 0.0, 1.0, 50.0, 0.0, out[i].ctypes.data)
    return out


def eval_camera_path(kfs, ts) -> np.ndarray:
    """CameraPath::eval_camera_path over the keyframe rows at each t: [n_t, 11]."""
    k = np.ascontiguousarray(kfs, np.float32).reshape(-1, 11)
    t = np.ascontiguousarray(ts, np.float32).reshape(-1)
    out = np.zeros((t.size, 11), np.float32)
    lib().refcam_eval(k.ctypes.data, k.shape[0], t.ctypes.data, t.size, out.ctypes.data)
    return out
