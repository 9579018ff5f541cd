"""ctypes wrapper of oracle/libmesh_opt_oracle.so (mesh_opt_oracle.cpp) — TEST INFRASTRUCTURE, like oracle.py.

The density input gradient and one mesh optimisation step on the CPU. The library also carries nerfshop_oracle.cpp (it includes it), so
the accumulator policy is set on it with its own orc_set_mlp_policy.
"""
from __future__ import annotations

import ctypes as C
import os
import shutil
import subprocess

import numpy as np

from . import oracle as orc

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmesh_opt_oracle.so")
_SOURCES = [os.path.join(_HERE, f) for f in ("mesh_opt_oracle.cpp", "nerfshop_oracle.cpp")] + [os.path.join(_HERE, "..", "include", "nerfshop_b200.h")]


def build(force: bool = False) -> str:
    """Compiles the library with the flags of oracle/Makefile (-ffp-contract=off: FMAs only where the source spells fmaf())."""
    if not force and os.path.exists(LIB_PATH) and all(os.path.getmtime(LIB_PATH) >= os.path.getmtime(s) for s in _SOURCES):
        return LIB_PATH
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else (shutil.which("g++") or "g++")
    cmd = [cxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-fopenmp", "-shared", "-o", LIB_PATH,
           os.path.join(_HERE, "mesh_opt_oracle.cpp")]
    subprocess.run(cmd, check=True, capture_output=True)
    return LIB_PATH


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        l = C.CDLL(LIB_PATH)
        vp = C.c_void_p
        l.orc_density_gradient.argtypes = [C.POINTER(orc.OrcScene), vp, C.c_uint32, vp, vp, vp, vp]
        l.orc_density_f64.argtypes = [C.POINTER(orc.OrcScene), vp, C.c_uint32, vp, vp]
        l.orc_mesh_opt_step.argtypes = [C.c_uint32, vp, vp, C.c_uint32, vp, vp, vp, vp, vp, vp, vp, vp]
        l.orc_mesh_opt_gradient.argtypes = [C.c_uint32, vp, vp, C.c_uint32, vp, vp, vp, vp, vp, vp]
        l.orc_adam_step.argtypes = [C.c_uint32, vp, vp, vp, vp, vp, vp]
        l.orc_set_mlp_policy.argtypes = [C.c_int]
        _lib = l
    return _lib


def _ptr(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def set_mlp_policy(policy: int) -> int:
    """1 = fp16 accumulation per k-chunk of 16 (default), 0 = wide; returns the old policy (nerfshop_oracle.cpp's orc_set_mlp_policy)."""
    return lib().orc_set_mlp_policy(policy)


def density_gradient(o: "orc.Oracle", coords: np.ndarray, dfeat: np.ndarray | None = None):
    """(grad float32 [n, 3], dfeat fp16 bits [32, n], raw density fp16 bits [n]) of NerfCoordinate rows; `dfeat` given: the grid
    backward of that feature gradient (fp16 bits [32, n]) instead of the MLP's."""
    c = np.ascontiguousarray(coords, np.float32)
    n = c.shape[0]
    din = None if dfeat is None else np.ascontiguousarray(dfeat, np.uint16)
    grad = np.zeros((n, 3), np.float32)
    df = np.zeros((32, n), np.uint16)
    dens = np.zeros(n, np.uint16)
    assert lib().orc_density_gradient(C.byref(o.scene), _ptr(c), n, _ptr(din), _ptr(grad), _ptr(df), _ptr(dens)) == 0
    return grad, df, dens


def density_f64(o: "orc.Oracle", pos: np.ndarray, want_grad: bool = True):
    """float64 without rounding: (raw density [n], analytic gradient [n, 3] or None) at warped positions [n, 3]."""
    p = np.ascontiguousarray(pos, np.float64)
    n = p.shape[0]
    dens = np.zeros(n, np.float64)
    grad = np.zeros((n, 3), np.float64) if want_grad else None
    assert lib().orc_density_f64(C.byref(o.scene), _ptr(p), n, _ptr(dens), _ptr(grad)) == 0
    return dens, grad


def mesh_opt_step(pos, faces, dens_fp16, grad, thresh, smooth_amount, density_amount, inflate_amount, state=None):
    """One step on all rows of pos [rows, 3] float32. state = (m1, m2, steps) arrays [rows, 3] (zeros when None), updated in place.
    Returns (new positions, normals of `pos`, state)."""
    pos = np.ascontiguousarray(pos, np.float32)
    rows = pos.shape[0]
    F = np.ascontiguousarray(faces, np.uint32).reshape(-1)
    if state is None:
        state = (np.zeros((rows, 3), np.float32), np.zeros((rows, 3), np.float32), np.zeros((rows, 3), np.uint32))
    k = np.array([thresh, smooth_amount, density_amount, inflate_amount], np.float32)
    out, nrm = np.zeros_like(pos), np.zeros_like(pos)
    d = np.ascontiguousarray(dens_fp16, np.uint16)
    g = np.ascontiguousarray(grad, np.float32)
    assert lib().orc_mesh_opt_step(rows, _ptr(pos), _ptr(F), F.size // 3, _ptr(d), _ptr(g), _ptr(k), _ptr(state[0]), _ptr(state[1]), _ptr(state[2]),
                                   _ptr(out), _ptr(nrm)) == 0
    return out, nrm, state


def mesh_opt_gradient(pos, faces, dens_fp16, grad, thresh, smooth_amount, density_amount, inflate_amount):
    """(1-ring sums [rows, 4], normals [rows, 3], opt gradient [rows, 3]) of compute_mesh_1ring + compute_mesh_opt_gradients_kernel."""
    pos = np.ascontiguousarray(pos, np.float32)
    rows = pos.shape[0]
    F = np.ascontiguousarray(faces, np.uint32).reshape(-1)
    k = np.array([thresh, smooth_amount, density_amount, inflate_amount], np.float32)
    sums, nrm, g = np.zeros((rows, 4), np.float32), np.zeros((rows, 3), np.float32), np.zeros((rows, 3), np.float32)
    assert lib().orc_mesh_opt_gradient(rows, _ptr(pos), _ptr(F), F.size // 3, _ptr(np.ascontiguousarray(dens_fp16, np.uint16)),
                                       _ptr(np.ascontiguousarray(grad, np.float32)), _ptr(k), _ptr(sums), _ptr(nrm), _ptr(g)) == 0
    return sums, nrm, g


def adam_step(x, g, state=None):
    """The restated tcnn Adam on the coordinates of x [rows, 3] with gradient g; state = (m1, m2, steps), zeros when None, updated in place."""
    x = np.ascontiguousarray(x, np.float32)
    g = np.ascontiguousarray(g, np.float32)
    if state is None:
        state = (np.zeros(x.shape, np.float32), np.zeros(x.shape, np.float32), np.zeros(x.shape, np.uint32))
    out = np.zeros_like(x)
    assert lib().orc_adam_step(x.size, _ptr(x), _ptr(g), _ptr(state[0]), _ptr(state[1]), _ptr(state[2]), _ptr(out)) == 0
    return out, state
