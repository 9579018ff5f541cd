"""ctypes wrapper of oracle/_ref/libnerfshop_ref_slices_cuda.so (oracle/ref_slices_build.py): the reference's slice-export code.
TEST INFRASTRUCTURE: only tests/ and tools/ import this. Host functions take and return numpy arrays; the *_dev functions take
CUDA tensors and run on the current stream."""
from __future__ import annotations

import ctypes as C
import os
import tempfile

import numpy as np

from . import ref_slices_build

_lib = None


def available() -> bool:
    return ref_slices_build.build() is not None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        path = ref_slices_build.build()
        if path is None:
            raise RuntimeError("oracle/_ref: no libnerfshop_ref_slices_cuda.so (the reference's sources are absent and none was built)")
        l = C.CDLL(path)
        V = C.c_void_p
        l.ref_slices_coordinate_floats.restype = C.c_uint32
        l.ref_slices_grid_coords.argtypes = [V, V, V, V, V, V]
        l.ref_slices_compute_nerf_density.argtypes = [C.c_uint32, V, C.c_int32, C.c_int32, V]
        l.ref_slices_density_png.argtypes = [V, V, C.c_float, C.c_int32, C.c_float, C.c_char_p]
        l.ref_slices_rgba_png.argtypes = [V, V, C.c_int32, C.c_char_p]
        l.ref_slices_n_records.restype = C.c_uint32
        l.ref_slices_record.argtypes = [C.c_uint32, C.c_char_p, C.c_uint32, V, V]
        l.ref_slices_info_text.restype = C.c_char_p
        _lib = l
    return _lib


def _f32(a):
    return np.ascontiguousarray(a, np.float32)


def _box(aabb):
    return _f32(np.concatenate([np.asarray(aabb[0], np.float32).reshape(3), np.asarray(aabb[1], np.float32).reshape(3)]))


def _ok(rc, what):
    if rc != 0:
        raise RuntimeError(f"reference {what} failed")


def _stream():
    import torch

    return torch.cuda.current_stream().cuda_stream


def grid_coords_dev(res, render_aabb, train_aabb, ray_dir, out):
    """generate_grid_samples_nerf_uniform_dir into `out` (float32 CUDA tensor of n x coordinate_floats): NerfCoordinate rows, x fastest."""
    r, rb, tb, d = np.asarray(res, np.int32), _box(render_aabb), _box(train_aabb), _f32(ray_dir)
    _ok(lib().ref_slices_grid_coords(r.ctypes.data, rb.ctypes.data, tb.ctypes.data, d.ctypes.data, out.data_ptr(), _stream()),
        "generate_grid_samples_nerf_uniform_dir")
    return out


def compute_nerf_density_dev(rgba, rgb_activation: int, density_activation: int):
    """compute_nerf_density in place on a float32 CUDA tensor of n x 4 network outputs."""
    _ok(lib().ref_slices_compute_nerf_density(rgba.shape[0], rgba.data_ptr(), int(rgb_activation), int(density_activation), _stream()),
        "compute_nerf_density")
    return rgba


def grid_coords(res, render_aabb, train_aabb, ray_dir) -> np.ndarray:
    """NerfCoordinate rows [n, coordinate_floats] of generate_grid_samples_nerf_uniform_dir."""
    import torch

    n = int(np.prod(np.asarray(res, np.int64)))
    out = torch.zeros((n, lib().ref_slices_coordinate_floats()), dtype=torch.float32, device="cuda")
    grid_coords_dev(res, render_aabb, train_aabb, ray_dir, out)
    return out.cpu().numpy()


def compute_nerf_density(rgbd, rgb_activation: int, density_activation: int) -> np.ndarray:
    """compute_nerf_density on network outputs rgbd [n, 4] (rgb, density as float)."""
    import torch

    t = torch.from_numpy(_f32(rgbd).copy()).cuda()
    compute_nerf_density_dev(t, rgb_activation, density_activation)
    return t.cpu().numpy()


def _records():
    out = []
    whc = np.zeros(3, np.int32)
    name = C.create_string_buffer(4096)
    for i in range(lib().ref_slices_n_records()):
        _ok(lib().ref_slices_record(i, name, len(name), whc.ctypes.data, None), "record")
        w, h, c = (int(v) for v in whc)
        px = np.zeros((h, w, c), np.uint8)
        _ok(lib().ref_slices_record(i, name, len(name), whc.ctypes.data, px.ctypes.data), "record")
        out.append((os.path.basename(name.value.decode()), px if c > 1 else px[:, :, 0]))
    lib().ref_slices_clear()
    return out


def density_png(density, res, thresh: float, swap_y_z: bool, density_range: float):
    """save_density_grid_to_png: (file name, pixels [h, w] uint8 as handed to stbi_write_png, counts int64 [2] as logged)."""
    d, r = _f32(density).reshape(-1), np.asarray(res, np.int32)
    lib().ref_slices_clear()
    _ok(lib().ref_slices_density_png(d.ctypes.data, r.ctypes.data, float(thresh), int(bool(swap_y_z)), float(density_range), b"ref"),
        "save_density_grid_to_png")
    text = lib().ref_slices_info_text().decode()
    (name, px), = _records()
    counts = np.array([int(text.split("#zero-x voxels=")[1].split()[0]), int(text.split("#lattice near zero-x=")[1].split()[0])], np.int64)
    return name, px, counts


def rgba_png(rgba, res, swap_y_z: bool):
    """save_rgba_grid_to_png_sequence: (file names, pixels [slices, h, w, 4] uint8), in z order."""
    x, r = _f32(rgba).reshape(-1), np.asarray(res, np.int32)
    lib().ref_slices_clear()
    with tempfile.TemporaryDirectory() as d:
        _ok(lib().ref_slices_rgba_png(x.ctypes.data, r.ctypes.data, int(bool(swap_y_z)), d.encode()), "save_rgba_grid_to_png_sequence")
    recs = _records()
    return [n for n, _ in recs], np.stack([p for _, p in recs])
