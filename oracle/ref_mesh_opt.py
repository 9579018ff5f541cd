"""ctypes wrapper of oracle/_ref/libnerfshop_ref_mesh_opt_cuda.so (oracle/ref_mesh_opt_build.py): the reference's mesh optimisation gradient
on the GPU. TEST INFRASTRUCTURE: only tests/ and tools/ import this. Every function takes and returns numpy arrays."""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import ref_mesh_opt_build

_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        path = ref_mesh_opt_build.build()
        if path is None:
            raise RuntimeError("oracle/_ref: no libnerfshop_ref_mesh_opt_cuda.so (the reference's sources are absent and none was built)")
        l = C.CDLL(path)
        V = C.c_void_p
        l.ref_mesh_opt_gradients.argtypes = [C.c_uint32, V, C.c_uint32, V, V, C.c_uint32, V, C.c_float, C.c_float, C.c_float, C.c_float, V, V, V]
        _lib = l
    return _lib


def opt_gradients(V, F, dens_fp16, input_gradients, thresh: float, smooth_amount: float, density_amount: float, inflate_amount: float):
    """compute_mesh_1ring + compute_mesh_opt_gradients on vertex rows V [n, 3] and faces F, with the fp16 density row dens_fp16 [n] (uint16 bits)
    and input_gradients [n, width] (the first 3 floats of a row are the position gradient): (opt gradient [n, 3], 1-ring sums [n, 4],
    normals [n, 3])."""
    v = np.ascontiguousarray(V, np.float32)
    f = np.ascontiguousarray(F, np.uint32)
    d = np.ascontiguousarray(dens_fp16, np.uint16)
    g = np.ascontiguousarray(input_gradients, np.float32)
    n = v.shape[0]
    grad, sums, nrm = np.zeros((n, 3), np.float32), np.zeros((n, 4), np.float32), np.zeros((n, 3), np.float32)
    rc = lib().ref_mesh_opt_gradients(n, v.ctypes.data, f.size, f.ctypes.data, d.ctypes.data, g.shape[1], g.ctypes.data, float(thresh), float(smooth_amount),
                                      float(density_amount), float(inflate_amount), grad.ctypes.data, sums.ctypes.data, nrm.ctypes.data)
    if rc != 0:
        raise RuntimeError("reference compute_mesh_opt_gradients failed")
    return grad, sums, nrm
