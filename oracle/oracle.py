"""ctypes wrapper of oracle/libnerfshop_oracle.so — TEST INFRASTRUCTURE (see nerfshop_oracle.cpp header).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs import this.
The struct layouts are the public ones of include/nerfshop_b200.h (imported from nerfshop_b200.abi, types only).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from nerfshop_b200 import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libnerfshop_oracle.so")


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "nerfshop_oracle.cpp")
    if force or not os.path.exists(LIB_PATH) or os.path.getmtime(LIB_PATH) < os.path.getmtime(src):
        subprocess.run(["make", "-C", _HERE, "-B" if force else "-s"], check=True, capture_output=True)
    return LIB_PATH


class OrcScene(C.Structure):
    _fields_ = [
        ("desc", abi.NsbModelDesc), ("params", C.c_void_p), ("n_params", C.c_uint64),
        ("bitfield", C.c_void_p), ("ops", C.POINTER(abi.NsbEditOp)), ("n_ops", C.c_int32),
    ]


class OrcStats(C.Structure):
    _fields_ = [
        ("n_rays", C.c_uint64), ("n_rays_alive", C.c_uint64), ("n_hit", C.c_uint64),
        ("n_samples", C.c_uint64), ("n_old_samples", C.c_uint64), ("threads", C.c_int32),
    ]


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        l = C.CDLL(LIB_PATH)
        l.orc_f2h.restype = C.c_uint16
        l.orc_f2h.argtypes = [C.c_float]
        l.orc_h2f.restype = C.c_float
        l.orc_h2f.argtypes = [C.c_uint16]
        l.orc_ld_random_val.restype = C.c_float
        l.orc_ld_random_val.argtypes = [C.c_uint32, C.c_uint32]
        l.orc_pixel_offset.argtypes = [C.c_uint32, C.c_void_p]
        l.orc_morton3D.restype = C.c_uint32
        l.orc_morton3D.argtypes = [C.c_uint32] * 3
        l.orc_mip_from_pos.argtypes = [C.c_float] * 3
        l.orc_cascaded_grid_idx_at.restype = C.c_uint32
        l.orc_cascaded_grid_idx_at.argtypes = [C.c_float] * 3 + [C.c_uint32]
        l.orc_model_n_params.argtypes = [C.POINTER(abi.NsbModelDesc), C.POINTER(C.c_uint64)]
        l.orc_level_table.argtypes = [C.POINTER(abi.NsbModelDesc)] + [C.c_void_p] * 4
        l.orc_grid_index.argtypes = [C.POINTER(abi.NsbModelDesc), C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p]
        l.orc_f2i.restype = C.c_int32
        l.orc_f2i.argtypes = [C.c_float]
        l.orc_encode.argtypes = [C.POINTER(OrcScene), C.c_void_p, C.c_uint32, C.c_void_p]
        l.orc_inference.argtypes = [C.POINTER(OrcScene), C.c_void_p, C.c_uint32, C.c_void_p, C.c_int]
        l.orc_map_rays.argtypes = [C.POINTER(OrcScene), C.c_void_p, C.c_void_p, C.c_uint32]
        l.orc_poisson_residuals.argtypes = [C.POINTER(OrcScene), C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        l.orc_map_positions.argtypes = [C.POINTER(OrcScene), C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
        l.orc_poisson_residual_density.argtypes = [C.POINTER(OrcScene), C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
        l.orc_march_trace.argtypes = [C.POINTER(OrcScene), C.POINTER(abi.NsbFrame), C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p]
        l.orc_render.argtypes = [C.POINTER(OrcScene), C.POINTER(abi.NsbFrame), C.c_void_p, C.c_void_p, C.POINTER(OrcStats), C.c_void_p]
        l.orc_set_threads.argtypes = [C.c_int]
        l.orc_set_mlp_policy.argtypes = [C.c_int]
        l.orc_density_grid_to_bitfield.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_float)]
        l.orc_pcg32_seed.argtypes = [C.c_uint64, C.c_uint64, C.c_void_p]
        l.orc_pcg32_seed.restype = None
        l.orc_pcg32_next.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
        l.orc_pcg32_next.restype = None
        l.orc_pcg32_advance.argtypes = [C.c_void_p, C.c_uint64]
        l.orc_pcg32_advance.restype = None
        l.orc_update_density_grid.argtypes = [C.POINTER(OrcScene), C.POINTER(abi.NsbGridUpdate), C.c_void_p, C.c_void_p, C.POINTER(C.c_float), C.c_void_p,
                                              C.c_void_p, C.c_void_p]
        l.orc_poisson_boundary.argtypes = [C.POINTER(OrcScene), C.c_void_p, C.c_uint32, C.POINTER(abi.NsbBoundarySampling), C.c_void_p, C.c_void_p, C.c_void_p]
        l.orc_poisson_boundary_ex.argtypes = [C.POINTER(OrcScene), C.c_void_p, C.c_uint32, C.POINTER(abi.NsbBoundarySampling), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        l.orc_membrane_blend.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 7
        l.orc_accumulate.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_float, C.c_int]
        l.orc_tonemap.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.POINTER(abi.NsbTonemap)]
        _lib = l
    return _lib


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


class Oracle:
    """Holds a scene (model params, occupancy bitfield, edit operators) for the CPU restatement."""

    def __init__(self, desc: abi.NsbModelDesc, params_u16: np.ndarray, bitfield: np.ndarray | None, ops=None):
        self.lib = lib()
        self.params = np.ascontiguousarray(params_u16, dtype=np.uint16)
        self.bitfield = None if bitfield is None else np.ascontiguousarray(bitfield, dtype=np.uint8)
        self.scene = OrcScene()
        self.scene.desc = desc
        self.scene.params = self.params.ctypes.data
        self.scene.n_params = self.params.size
        self.scene.bitfield = None if self.bitfield is None else self.bitfield.ctypes.data
        self.set_ops(ops)

    def set_ops(self, ops):
        """ops: list of (NsbEditOp, keepalive) or None. The structs hold host pointers into keepalive arrays."""
        self._ops_keep = ops
        if ops:
            arr = (abi.NsbEditOp * len(ops))(*[o[0] for o in ops])
            self._ops_arr = arr
            self.scene.ops = C.cast(arr, C.POINTER(abi.NsbEditOp))
            self.scene.n_ops = len(ops)
        else:
            self.scene.ops = None
            self.scene.n_ops = 0

    def encode(self, coords: np.ndarray) -> np.ndarray:
        coords = np.ascontiguousarray(coords, np.float32)
        n = coords.shape[0]
        out = np.zeros((32, n), np.uint16)
        assert self.lib.orc_encode(C.byref(self.scene), _ptr(coords), n, _ptr(out)) == 0
        return out

    def inference(self, coords: np.ndarray, density_only: bool = False) -> np.ndarray:
        coords = np.ascontiguousarray(coords, np.float32)
        n = coords.shape[0]
        out = np.zeros((16, n), np.uint16)
        assert self.lib.orc_inference(C.byref(self.scene), _ptr(coords), n, _ptr(out), int(density_only)) == 0
        return out

    def map_rays(self, coords: np.ndarray):
        c = np.ascontiguousarray(coords, np.float32).copy()
        mask = np.zeros(c.shape[0], np.uint8)
        assert self.lib.orc_map_rays(C.byref(self.scene), _ptr(c), _ptr(mask), c.shape[0]) == 0
        return c, mask

    def poisson_residuals(self, coords: np.ndarray):
        c = np.ascontiguousarray(coords, np.float32)
        n = c.shape[0]
        sh = np.zeros((n, 27), np.float32)
        od = np.zeros(n, np.float32)
        rd = np.zeros(n, np.float32)
        assert self.lib.orc_poisson_residuals(C.byref(self.scene), _ptr(c), n, _ptr(sh), _ptr(od), _ptr(rd)) == 0
        return sh, od, rd

    def map_positions(self, positions: np.ndarray, mask: np.ndarray | None = None):
        """EditOperator::map_positions over all operators. positions: float32 [n, stride >= 3], warped position in the first 3 columns
        (mapped in place on a copy). mask: uint8 [n] that the operators may only set, or None. Returns (positions, mask)."""
        p = np.ascontiguousarray(positions, np.float32).copy()
        m = None if mask is None else np.ascontiguousarray(mask, np.uint8).copy()
        assert self.lib.orc_map_positions(C.byref(self.scene), _ptr(p), p.shape[1], None if m is None else _ptr(m), p.shape[0]) == 0
        return p, m

    def poisson_residual_density(self, positions: np.ndarray, density_fp16: np.ndarray) -> np.ndarray:
        """EditOperator::compute_poisson_residual_density over all operators: density_fp16 (uint16 bits [n]) plus the residuals at positions [n, stride]."""
        p = np.ascontiguousarray(positions, np.float32)
        h = np.ascontiguousarray(density_fp16).view(np.uint16).copy()
        assert self.lib.orc_poisson_residual_density(C.byref(self.scene), _ptr(p), p.shape[1], _ptr(h), p.shape[0]) == 0
        return h

    def march_trace(self, frame: abi.NsbFrame, pixels: np.ndarray, max_samples: int):
        pixels = np.ascontiguousarray(pixels, np.uint32)
        n = pixels.size
        rec = np.zeros((n, max_samples, 5), np.float32)
        idx = np.zeros((n, max_samples, 2), np.uint32)
        cnt = np.zeros(n, np.uint32)
        assert self.lib.orc_march_trace(C.byref(self.scene), C.byref(frame), _ptr(pixels), n, max_samples, _ptr(rec), _ptr(idx), _ptr(cnt)) == 0
        return rec, idx, cnt

    def update_density_grid(self, params: "abi.NsbGridUpdate", grid: np.ndarray, want_samples: bool = False, want_splats: bool = False):
        """Testbed::update_density_grid_nerf_operator on the host. Returns (grid, bitfield, mean[, samples][, splats]).
        samples: float32 [n, 4] {mapped warped position, activated + residual density}. splats: (cell uint32 [n], the sample's splat
        cell; residual uint16 [n], the fp16 bits of the membrane residual added to its activated density: 0 if none, NaN if several)."""
        grid = np.ascontiguousarray(grid, np.float32).reshape(-1).copy()
        bits = np.zeros(abi.NSB_BITFIELD_BYTES, np.uint8)
        mean = C.c_float()
        n = params.n_uniform_samples + params.n_nonuniform_samples
        samples = np.zeros((n, 4), np.float32) if want_samples else None
        cells = np.zeros(n, np.uint32) if want_splats else None
        residual = np.zeros(n, np.uint16) if want_splats else None
        rc = self.lib.orc_update_density_grid(C.byref(self.scene), C.byref(params), _ptr(grid), _ptr(bits), C.byref(mean),
                                              *[None if a is None else _ptr(a) for a in (samples, cells, residual)])
        assert rc == 0
        return (grid, bits, mean.value) + ((samples,) if want_samples else ()) + (((cells, residual),) if want_splats else ())

    def poisson_boundary_with_jitter(self, points: np.ndarray, params: "abi.NsbBoundarySampling", uniforms: np.ndarray):
        """compute_poisson_boundary with the jitter given (2 uniforms per sample, (vertex, i, j) order) instead of drawn from pcg32: (density, shs, coords)."""
        pts = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
        n = pts.shape[0]
        u = np.ascontiguousarray(uniforms, np.float32).reshape(-1)
        assert u.size == 2 * n * params.sampling_width ** 2
        dens, shs = np.zeros(n, np.float32), np.zeros((n, 27), np.float32)
        coords = np.zeros((n * params.sampling_width ** 2, 7), np.float32)
        assert self.lib.orc_poisson_boundary_ex(C.byref(self.scene), _ptr(pts), n, C.byref(params), _ptr(u), _ptr(dens), _ptr(shs), _ptr(coords)) == 0
        return dens, shs, coords

    def poisson_boundary(self, points: np.ndarray, params: "abi.NsbBoundarySampling", want_coords: bool = False):
        """GrowingSelection::compute_poisson_boundary: (density [n], shs [n, 27][, coords])."""
        pts = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
        n = pts.shape[0]
        dens, shs = np.zeros(n, np.float32), np.zeros((n, 27), np.float32)
        coords = np.zeros((n * params.sampling_width ** 2, 7), np.float32) if want_coords else None
        assert self.lib.orc_poisson_boundary(C.byref(self.scene), _ptr(pts), n, C.byref(params), _ptr(dens), _ptr(shs), None if coords is None else _ptr(coords)) == 0
        return (dens, shs, coords) if want_coords else (dens, shs)

    def render(self, frame: abi.NsbFrame, background: np.ndarray | None = None, want_margin: bool = False):
        W, H = frame.width, frame.height
        fb = np.zeros((H, W, 4), np.float32) if background is None else np.ascontiguousarray(background, np.float32).copy()
        depth = np.zeros((H, W), np.float32)
        margin = np.zeros((H, W), np.float32) if want_margin else None
        stats = OrcStats()
        rc = self.lib.orc_render(C.byref(self.scene), C.byref(frame), _ptr(fb), _ptr(depth), C.byref(stats), None if margin is None else _ptr(margin))
        assert rc == 0
        return fb, depth, stats, margin


def pcg32_seed(initstate: int, initseq: int):
    st = np.zeros(2, np.uint64)
    lib().orc_pcg32_seed(initstate, initseq, _ptr(st))
    return st


def pcg32_next(st: np.ndarray, n: int) -> np.ndarray:
    out = np.zeros(n, np.uint32)
    lib().orc_pcg32_next(_ptr(st), n, _ptr(out))
    return out


def pcg32_advance(st: np.ndarray, delta: int) -> None:
    lib().orc_pcg32_advance(_ptr(st), delta)


def membrane_blend(gamma, inside_density, outside_density, inside_shs, outside_shs):
    """GrowingSelection::interpolate_poisson_boundary: (boundary_shs [nv, 27], outside_density [nv], residual_density [nv])."""
    g = np.ascontiguousarray(gamma, np.float32)
    nv, ncv = g.shape
    arrs = [np.ascontiguousarray(a, np.float32) for a in (inside_density, outside_density, inside_shs, outside_shs)]
    b_shs, b_od, b_rd = np.zeros((nv, 27), np.float32), np.zeros(nv, np.float32), np.zeros(nv, np.float32)
    assert lib().orc_membrane_blend(_ptr(g), nv, ncv, *[_ptr(a) for a in arrs], _ptr(b_shs), _ptr(b_od), _ptr(b_rd)) == 0
    return b_shs, b_od, b_rd


def accumulate(frame: np.ndarray, acc: np.ndarray, spp: int, color_space: int = 0) -> np.ndarray:
    frame = np.ascontiguousarray(frame, np.float32)
    acc = np.zeros_like(frame) if spp == 0 else np.ascontiguousarray(acc, np.float32).copy()
    assert lib().orc_accumulate(_ptr(frame), _ptr(acc), frame.size // 4, float(spp), color_space) == 0
    return acc


def tonemap(acc: np.ndarray, params: "abi.NsbTonemap") -> np.ndarray:
    acc = np.ascontiguousarray(acc, np.float32)
    out = np.zeros_like(acc)
    assert lib().orc_tonemap(_ptr(acc), _ptr(out), acc.size // 4, C.byref(params)) == 0
    return out


def density_grid_to_bitfield(grid: np.ndarray):
    grid = np.ascontiguousarray(grid, np.float32).reshape(-1)
    bits = np.zeros(abi.NSB_BITFIELD_BYTES, np.uint8)
    mean = C.c_float()
    assert lib().orc_density_grid_to_bitfield(_ptr(grid), _ptr(bits), C.byref(mean)) == 0
    return bits, mean.value


def set_mlp_policy(policy: int) -> int:
    """1 = wmma __half accumulator fragments (round to fp16 after every k-chunk of 16; default), 0 = wide accumulate. Returns the old policy."""
    return lib().orc_set_mlp_policy(policy)


def set_threads(n: int) -> int:
    return lib().orc_set_threads(n)
