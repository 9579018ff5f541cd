"""Density and RGBA slices: the reference's PNG exports on top of the C ABI (nsb_density_on_grid, nsb_density_png, nsb_rgba_on_grid,
nsb_rgba_png). The pixels are computed on the device; only the finished images come back to the host.

  write_png                          <- stbi_write_png (8-bit grey or RGBA; a valid PNG of the same pixels, not stb's bytes)
  compute_and_save_png_slices        <- Testbed::compute_and_save_png_slices (testbed.cu:345-366) + save_density_grid_to_png
                                        (marching_cubes.cu:898-974), the GUI's "Save density PNG" (testbed.cu:952-954)
  get_rgba_on_grid                   <- Testbed::get_rgba_on_grid (testbed_nerf.cu:4588-4612)
  save_rgba_grid_to_png_sequence     <- save_rgba_grid_to_png_sequence (marching_cubes.cu:979-1015)
  compute_and_save_rgba_png_sequence <- the GUI's "Save RGBA PNG sequence" (testbed.cu:956-966)
"""
from __future__ import annotations

import ctypes as C
import os
import struct
import zlib

import numpy as np

from . import abi
from .mesh import get_marching_cubes_res


def density_png_extent(res3d, swap_y_z: bool = False):
    """(w, h) of save_density_grid_to_png's mosaic for a res3d grid (nsb_density_png_extent; needs no GPU)."""
    lib = abi.load_library()
    res = (C.c_int32 * 3)(*[int(v) for v in res3d])
    w, h = C.c_uint32(), C.c_uint32()
    abi.check(lib, lib.nsb_density_png_extent(res, int(bool(swap_y_z)), C.byref(w), C.byref(h)), "nsb_density_png_extent")
    return w.value, h.value


def _chunk(tag: bytes, data: bytes) -> bytes:
    return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)


def write_png(path: str, pixels, channels: int) -> None:
    """Writes uint8 pixels [h, w] (channels 1, grey) or [h, w, 4] (channels 4, RGBA) as an 8-bit PNG, every row unfiltered."""
    if channels not in (1, 4):
        raise ValueError("write_png: channels must be 1 (grey) or 4 (RGBA)")
    p = np.ascontiguousarray(np.asarray(pixels, np.uint8))
    h, w = p.shape[0], p.shape[1]
    if p.size != h * w * channels:
        raise ValueError(f"write_png: {p.shape} is not [h, w] x {channels} channel(s)")
    rows = p.reshape(h, w * channels)
    raw = np.zeros((h, w * channels + 1), np.uint8)  # filter byte 0 (None) before each row
    raw[:, 1:] = rows
    ihdr = struct.pack(">IIBBBBB", w, h, 8, 0 if channels == 1 else 6, 0, 0, 0)
    with open(path, "wb") as fh:
        fh.write(b"\x89PNG\r\n\x1a\n" + _chunk(b"IHDR", ihdr) + _chunk(b"IDAT", zlib.compress(raw.tobytes(), 6)) + _chunk(b"IEND", b""))


def compute_and_save_png_slices(renderer, filename: str, res: int, aabb, train_aabb, thresh: float = 2.5, density_range: float = 4.0,
                                flip_y_and_z_axes: bool = False):
    """The density of the field over `aabb` at get_marching_cubes_res(res, aabb), as one 8-bit mosaic of its z slices (y and z swapped when
    flip_y_and_z_axes) written to filename + ".density_slices_<x>x<y>x<z>.png" with the grid's resolution before the swap. Returns
    (res3d, counts): counts = (#zero-x voxels, #lattice near zero-x), the numbers the reference logs. The reference substitutes its
    m_mesh.thresh for a negative thresh and its m_render_aabb for an empty aabb; here both are used as given. The renderer needs a model
    and a running density grid (cells where it is empty read -10000, as in the reference)."""
    res3d = get_marching_cubes_res(res, aabb)
    density = renderer.density_on_grid(res3d, aabb, train_aabb)
    pixels, counts = renderer.density_png(density, res3d, thresh, density_range, flip_y_and_z_axes)
    write_png(filename + ".density_slices_%dx%dx%d.png" % tuple(int(v) for v in res3d), pixels.cpu().numpy(), 1)
    return res3d, tuple(int(v) for v in counts.cpu().tolist())


def get_rgba_on_grid(renderer, res3d, ray_dir, render_aabb, train_aabb, rgb_activation: int = abi.NSB_ACT_LOGISTIC,
                     density_activation: int = abi.NSB_ACT_EXPONENTIAL):
    """float32 CUDA tensor [res_z, res_y, res_x, 4]: premultiplied rgb and alpha of the field seen from ray_dir (NerfRenderer.rgba_on_grid)."""
    return renderer.rgba_on_grid(res3d, render_aabb, train_aabb, ray_dir, rgb_activation, density_activation)


def save_rgba_grid_to_png_sequence(renderer, rgba, path: str, res3d, flip_y_and_z_axes: bool = False) -> list:
    """Writes one RGBA PNG per z slice of `rgba` (y and z swapped when flip_y_and_z_axes) as path/%04d_<w>x<h>.png; returns the file names."""
    pixels = renderer.rgba_png(rgba, res3d, flip_y_and_z_axes).cpu().numpy()
    names = []
    for z in range(pixels.shape[0]):
        name = os.path.join(path, "%04d_%dx%d.png" % (z, pixels.shape[2], pixels.shape[1]))
        write_png(name, pixels[z], 4)
        names.append(name)
    return names


def compute_and_save_rgba_png_sequence(renderer, data_path: str, res: int, render_aabb, train_aabb, rgb_activation: int = abi.NSB_ACT_LOGISTIC,
                                       density_activation: int = abi.NSB_ACT_EXPONENTIAL, flip_y_and_z_axes: bool = False) -> list:
    """The GUI's "Save RGBA PNG sequence": the field over render_aabb at get_marching_cubes_res(res, render_aabb), seen along +y when the
    axes are swapped and +z otherwise, written to data_path/rgba_slices/ (created if missing). Returns the file names."""
    res3d = get_marching_cubes_res(res, render_aabb)
    ray_dir = (0.0, 1.0, 0.0) if flip_y_and_z_axes else (0.0, 0.0, 1.0)
    rgba = get_rgba_on_grid(renderer, res3d, ray_dir, render_aabb, train_aabb, rgb_activation, density_activation)
    out = os.path.join(data_path, "rgba_slices")
    if not os.path.isdir(out):
        os.mkdir(out)
    return save_rgba_grid_to_png_sequence(renderer, rgba, out, res3d, flip_y_and_z_axes)
