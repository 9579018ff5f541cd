"""ctypes wrapper of oracle/_ref/libnerfshop_ref_mesh_cuda.so (oracle/ref_mesh_build.py): the reference's mesh-extraction code on the
GPU. TEST INFRASTRUCTURE: only tests/ and tools/ import this. Every function takes and returns numpy arrays."""
from __future__ import annotations

import ctypes as C
import os
import tempfile

import numpy as np

from . import ref_mesh_build

_lib = None


def available() -> bool:
    return ref_mesh_build.build() is not None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        path = ref_mesh_build.build()
        if path is None:
            raise RuntimeError("oracle/_ref: no libnerfshop_ref_mesh_cuda.so (the reference's sources are absent and none was built)")
        l = C.CDLL(path)
        V = C.c_void_p
        l.ref_mesh_position_floats.restype = C.c_uint32
        l.ref_mesh_coordinate_floats.restype = C.c_uint32
        l.ref_mesh_res.argtypes = [C.c_uint32, V, V]
        l.ref_mesh_grid_positions.argtypes = [V, V, V, V]
        l.ref_mesh_half_to_float.argtypes = [C.c_uint32, V, V, V, V, V]
        l.ref_mesh_marching_cubes.argtypes = [V, V, C.c_float, V, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_float)]
        l.ref_mesh_get.argtypes = [V, V]
        l.ref_mesh_normals.argtypes = [C.c_uint32, V, C.c_uint32, V, V]
        l.ref_mesh_color_inputs.argtypes = [C.c_uint32, V, V, V]
        l.ref_mesh_srgb.argtypes = [C.c_uint32, V, C.c_int32, C.c_int32, V]
        l.ref_mesh_save.argtypes = [C.c_char_p, C.c_uint32, V, V, V, C.c_uint32, V, C.c_float, V]
        _lib = l
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def _box(aabb):
    """A [min, max] pair as 6 contiguous floats; the caller keeps the array alive across the call that reads its address."""
    return _f32(np.concatenate([np.asarray(aabb[0], np.float32).reshape(3), np.asarray(aabb[1], np.float32).reshape(3)]))


def _ok(rc, what):
    if rc != 0:
        raise RuntimeError(f"reference {what} failed")


def get_marching_cubes_res(res_1d: int, aabb) -> np.ndarray:
    out, box = np.zeros(3, np.int32), _box(aabb)
    _ok(lib().ref_mesh_res(int(res_1d), box.ctypes.data, out.ctypes.data), "get_marching_cubes_res")
    return out


def grid_positions(res, render_aabb, train_aabb, rows=None) -> np.ndarray:
    """generate_grid_samples_nerf_uniform: NerfPosition rows [n, position_floats] (x fastest); only the given point indices when rows is
    given (the kernel still runs on the whole grid)."""
    r = np.asarray(res, np.int32)
    out = np.zeros((int(np.prod(r.astype(np.int64))), lib().ref_mesh_position_floats()), np.float32)
    rb, tb = _box(render_aabb), _box(train_aabb)
    _ok(lib().ref_mesh_grid_positions(r.ctypes.data, rb.ctypes.data, tb.ctypes.data, out.ctypes.data), "generate_grid_samples_nerf_uniform")
    return out if rows is None else out[np.asarray(rows, np.int64)]


def half_to_float(positions, mlp_u16, train_aabb, density_grid=None) -> np.ndarray:
    """grid_samples_half_to_float: the filter is active when density_grid (float[5*128^3]) is given."""
    pos = _f32(positions)
    m = np.ascontiguousarray(mlp_u16, np.uint16)
    out = np.zeros(pos.shape[0], np.float32)
    g = None if density_grid is None else _f32(density_grid)
    tb = _box(train_aabb)
    _ok(lib().ref_mesh_half_to_float(pos.shape[0], tb.ctypes.data, m.ctypes.data, pos.ctypes.data,
                                     None if g is None else g.ctypes.data, out.ctypes.data), "grid_samples_half_to_float")
    return out


def marching_cubes(density, res, aabb, thresh: float, want_ms: bool = False):
    """marching_cubes_gpu: (V [rows, 3] with rows = vertices rounded up to 128, F [n_triangles, 3]) in the reference's atomic order."""
    r = np.asarray(res, np.int32)
    d = _f32(density).reshape(-1)
    nr, ni, ms = C.c_uint64(), C.c_uint64(), C.c_float()
    box = _box(aabb)
    _ok(lib().ref_mesh_marching_cubes(box.ctypes.data, r.ctypes.data, float(thresh), d.ctypes.data, C.byref(nr), C.byref(ni),
                                      C.byref(ms)), "marching_cubes_gpu")
    V = np.zeros((nr.value, 3), np.float32)
    F = np.zeros((ni.value // 3, 3), np.uint32)
    _ok(lib().ref_mesh_get(V.ctypes.data, F.ctypes.data), "marching_cubes_gpu download")
    return (V, F, ms.value) if want_ms else (V, F)


def normals(V, F) -> np.ndarray:
    """compute_mesh_1ring's vertex normals (area-weighted sums, not normalised) of the given mesh."""
    v, f = _f32(V), np.ascontiguousarray(F, np.uint32)
    out = np.zeros_like(v)
    _ok(lib().ref_mesh_normals(v.shape[0], v.ctypes.data, f.size, f.ctypes.data, out.ctypes.data), "compute_mesh_1ring")
    return out


def color_inputs(V, train_aabb) -> np.ndarray:
    """generate_nerf_network_inputs_from_positions: NerfCoordinate rows [n, coordinate_floats]."""
    v = _f32(V)
    out = np.zeros((v.shape[0], lib().ref_mesh_coordinate_floats()), np.float32)
    tb = _box(train_aabb)
    _ok(lib().ref_mesh_color_inputs(v.shape[0], tb.ctypes.data, v.ctypes.data, out.ctypes.data),
        "generate_nerf_network_inputs_from_positions")
    return out


def srgb(rgbd, rgb_activation: int, linear_colors: bool) -> np.ndarray:
    """extract_srgb_with_activation on network outputs rgbd [n, 4]."""
    x = _f32(rgbd)
    out = np.zeros((x.shape[0], 3), np.float32)
    _ok(lib().ref_mesh_srgb(x.shape[0], x.ctypes.data, int(rgb_activation), int(bool(linear_colors)), out.ctypes.data), "extract_srgb_with_activation")
    return out


def save_mesh(ext: str, V, N, Cc, F, nerf_scale: float, nerf_offset) -> np.ndarray:
    """The bytes save_mesh writes for a file name ending in `ext` (uint8 array)."""
    v, n, c, f, off = _f32(V), _f32(N), _f32(Cc), np.ascontiguousarray(F, np.uint32), _f32(nerf_offset)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "mesh" + ext)
        _ok(lib().ref_mesh_save(path.encode(), v.shape[0], v.ctypes.data, n.ctypes.data, c.ctypes.data, f.size, f.ctypes.data, float(nerf_scale),
                                off.ctypes.data), "save_mesh")
        with open(path, "rb") as fh:
            return np.frombuffer(fh.read(), np.uint8).copy()
