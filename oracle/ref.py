"""ctypes wrapper of oracle/_ref/libnerfshop_ref.so — the reference's own render-path sources compiled for the CPU
(oracle/ref_build.py, oracle/ref_driver.cpp). TEST INFRASTRUCTURE: only tests/ import this; it pins oracle/ to the reference.

The library is built where /root/reference exists (this container) and travels to the GPU box as a git-ignored .so.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from nerfshop_b200 import abi

from . import ref_build

INFER_FN = C.CFUNCTYPE(None, C.c_void_p, C.POINTER(C.c_float), C.c_uint32, C.POINTER(C.c_uint16))
_lib = None


def available() -> bool:
    return ref_build.build() is not None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        path = ref_build.build()
        if path is None:
            raise RuntimeError("oracle/_ref: /root/reference is absent and no prebuilt libnerfshop_ref.so travelled with the repo")
        l = C.CDLL(path)
        V = C.c_void_p
        l.ref_ld_random_val.argtypes = [C.c_uint32, V, V, V]
        l.ref_ld_random_pixel_offset.argtypes = [C.c_uint32, V]
        l.ref_morton3D.argtypes = [C.c_uint32, V, V]
        l.ref_mip.argtypes = [C.c_uint32, V, V, V, V, V]
        l.ref_calc_dt.argtypes = [C.c_uint32, V, C.c_float, V]
        l.ref_advance_to_next_voxel.argtypes = [C.c_uint32, V, C.c_float, V, V, V, V]
        l.ref_warp.argtypes = [C.c_uint32, V, V, V, V, V, V, V]
        l.ref_ray_intersect.argtypes = [C.c_uint32, V, V, V, V, V, V]
        l.ref_srgb_to_linear.argtypes = [C.c_uint32, V, V]
        l.ref_evaluate_sh9.argtypes = [C.c_uint32, V, V, V]
        l.ref_activations.argtypes = [C.c_uint32, V, C.c_int, V, V]
        l.ref_pcg32.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32, V, V]
        l.ref_grid_samples.argtypes = [C.c_uint32, C.c_uint64, C.c_uint64, C.c_uint32, V, V, V, C.c_uint32, C.c_float, V, V]
        l.ref_march_trace.argtypes = [C.POINTER(abi.NsbFrame), V, V, C.c_uint32, C.c_uint32, V, V, V, V]
        l.ref_render.argtypes = [C.POINTER(abi.NsbFrame), V, C.POINTER(abi.NsbEditOp), C.c_int, INFER_FN, V, V, V, V]
        l.ref_map_rays.argtypes = [C.POINTER(abi.NsbEditOp), C.c_int, V, V, C.c_uint32]
        l.ref_poisson_residuals.argtypes = [C.POINTER(abi.NsbEditOp), C.c_int, V, C.c_uint32, V, V, V]
        l.ref_compute_mvc.argtypes = [V, C.c_uint32, V, C.c_uint32, V, C.c_uint32, V, C.c_float, C.c_int]
        l.ref_tet_mesh_build.argtypes = [V, V, C.c_uint32, V, C.c_uint32, V, V, V, V, V, C.c_uint32, V, V, V]
        l.ref_svd3.argtypes = [C.c_uint32, V, V]
        l.ref_set_parallel.argtypes = [C.c_int]
        _lib = l
    return _lib


# entry points added to ref_driver.cpp after libraries that may still be in use were built: where the reference's sources are absent, a
# prebuilt library is used as it is and may lack them
_LATER = {"map_positions": "ref_map_positions", "poisson_residual_density": "ref_poisson_residual_density"}


def serves(name: str) -> bool:
    """The loaded library has the entry point behind this module's function `name`."""
    return name not in _LATER or hasattr(lib(), _LATER[name])


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def f32(a):
    return np.ascontiguousarray(a, np.float32)


def u32(a):
    return np.ascontiguousarray(a, np.uint32)


def ld_random_val(index, seed):
    index, seed = u32(index), u32(seed)
    out = np.zeros(index.size, np.float32)
    lib().ref_ld_random_val(index.size, _p(index), _p(seed), _p(out))
    return out


def ld_random_pixel_offset(spp: int):
    out = np.zeros(2, np.float32)
    lib().ref_ld_random_pixel_offset(spp, _p(out))
    return out


def morton3D(xyz):
    xyz = u32(xyz)
    out = np.zeros(xyz.shape[0], np.uint32)
    lib().ref_morton3D(xyz.shape[0], _p(xyz), _p(out))
    return out


def mip(pos, dt):
    pos, dt = f32(pos), f32(dt)
    n = pos.shape[0]
    mp, md, cell = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.uint32)
    lib().ref_mip(n, _p(pos), _p(dt), _p(mp), _p(md), _p(cell))
    return mp, md, cell


def calc_dt(t, cone):
    t = f32(t)
    out = np.zeros_like(t)
    lib().ref_calc_dt(t.size, _p(t), cone, _p(out))
    return out


def advance_to_next_voxel(t, cone, pos, dirs, res):
    t, pos, dirs, res = f32(t), f32(pos), f32(dirs), u32(res)
    out = np.zeros_like(t)
    lib().ref_advance_to_next_voxel(t.size, _p(t), cone, _p(pos), _p(dirs), _p(res), _p(out))
    return out


def warp(pos, dirs, dt, amin, amax):
    pos, dirs, dt, amin, amax = f32(pos), f32(dirs), f32(dt), f32(amin), f32(amax)
    n = pos.shape[0]
    out, back = np.zeros((n, 7), np.float32), np.zeros((n, 7), np.float32)
    lib().ref_warp(n, _p(pos), _p(dirs), _p(dt), _p(amin), _p(amax), _p(out), _p(back))
    return out, back


def ray_intersect(o, d, mn, mx):
    o, d, mn, mx = f32(o), f32(d), f32(mn), f32(mx)
    n = o.shape[0]
    t, c = np.zeros(n, np.float32), np.zeros(n, np.uint8)
    lib().ref_ray_intersect(n, _p(o), _p(d), _p(mn), _p(mx), _p(t), _p(c))
    return t, c


def srgb_to_linear(x):
    x = f32(x)
    out = np.zeros_like(x)
    lib().ref_srgb_to_linear(x.size, _p(x), _p(out))
    return out


def evaluate_sh9(sh, dirs):
    sh, dirs = f32(sh), f32(dirs)
    out = np.zeros((dirs.shape[0], 3), np.float32)
    lib().ref_evaluate_sh9(dirs.shape[0], _p(sh), _p(dirs), _p(out))
    return out


def activations(x, act: int):
    x = f32(x)
    rgb, dens = np.zeros_like(x), np.zeros_like(x)
    lib().ref_activations(x.size, _p(x), act, _p(rgb), _p(dens))
    return rgb, dens


def pcg32(initstate: int, initseq: int, advance: int, n: int):
    u, f = np.zeros(n, np.uint32), np.zeros(n, np.float32)
    lib().ref_pcg32(initstate, initseq, advance, n, _p(u), _p(f))
    return u, f


def grid_samples(n, rng_state, rng_inc, step, amin, amax, grid, n_cascades, thresh):
    amin, amax, grid = f32(amin), f32(amax), f32(grid)
    pos, idx = np.zeros((n, 3), np.float32), np.zeros(n, np.uint32)
    lib().ref_grid_samples(n, rng_state, rng_inc, step, _p(amin), _p(amax), _p(grid), n_cascades, thresh, _p(pos), _p(idx))
    return pos, idx


def grid_to_bitfield(grid, mean: float):
    """grid_to_bitfield + bitfield_max_pool (testbed_nerf.cu:514-555) as update_density_grid_mean_and_bitfield launches them."""
    grid = f32(grid)
    bits = np.zeros(abi.NSB_BITFIELD_BYTES, np.uint8)
    lib().ref_grid_to_bitfield.argtypes = [C.c_void_p, C.c_float, C.c_void_p]
    lib().ref_grid_to_bitfield(_p(grid), float(mean), _p(bits))
    return bits


def update_density_grid(params: "abi.NsbGridUpdate", grid, density, ops=None):
    """Testbed::update_density_grid_nerf_operator + update_density_grid_mean_and_bitfield of the reference (testbed_nerf.cu:3533-3658).
    density(positions [n, 3] float32, warped) -> [16, n] uint16 (fp16 bits, row 0 = raw density) is NerfNetwork::density.
    Returns (grid, bitfield, mean)."""
    grid = f32(grid).reshape(-1).copy()
    bits = np.zeros(abi.NSB_BITFIELD_BYTES, np.uint8)
    mean = C.c_float()

    def cb(_user, pos_p, n, out_p):
        pos = np.ctypeslib.as_array(pos_p, shape=(n, 3))
        np.ctypeslib.as_array(out_p, shape=(16, n))[:] = density(pos)

    fn = INFER_FN(cb)
    arr, n_ops = _ops_array(ops)
    l = lib()
    l.ref_update_density_grid.argtypes = [C.POINTER(abi.NsbGridUpdate), C.POINTER(abi.NsbEditOp), C.c_int, INFER_FN, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_float)]
    rc = l.ref_update_density_grid(C.byref(params), arr, n_ops, fn, None, _p(grid), _p(bits), C.byref(mean))
    assert rc == 0
    return grid, bits, mean.value


def accumulate(frame, acc, sample_count: float, color_space: int):
    """accumulate_kernel (render_buffer.cu:217-252): returns the new accumulate buffer."""
    frame, acc = f32(frame), f32(acc).copy()
    H, W = frame.shape[:2]
    l = lib()
    l.ref_accumulate.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_float, C.c_int]
    assert l.ref_accumulate(W, H, _p(frame), _p(acc), float(sample_count), int(color_space)) == 0
    return acc


def tonemap(acc, exposure: float, background, color_space: int, output_color_space: int, curve: int, clamp_output: bool):
    """tonemap_kernel (render_buffer.cu:471-501) and the two tonemap() device functions (:254-332)."""
    acc, bg = f32(acc), f32(background)
    H, W = acc.shape[:2]
    out = np.zeros_like(acc)
    l = lib()
    l.ref_tonemap.argtypes = [C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    assert l.ref_tonemap(W, H, float(exposure), _p(bg), _p(acc), int(color_space), int(output_color_space), int(curve), int(bool(clamp_output)), _p(out)) == 0
    return out


def membrane_blend(gamma, inside_density, outside_density, inside_shs, outside_shs):
    """The loop of GrowingSelection::interpolate_poisson_boundary (growing_selection.cu:2363-2392): (boundary_shs [nv, 27], outside_density, residual_density)."""
    g = f32(gamma)
    nv, ncv = g.shape
    arrs = [f32(a) for a in (inside_density, outside_density, inside_shs, outside_shs)]
    b_shs, b_od, b_rd = np.zeros((nv, 27), np.float32), np.zeros(nv, np.float32), np.zeros(nv, np.float32)
    l = lib()
    l.ref_membrane_blend.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32] + [C.c_void_p] * 7
    assert l.ref_membrane_blend(_p(g), nv, ncv, *[_p(a) for a in arrs], _p(b_shs), _p(b_od), _p(b_rd)) == 0
    return b_shs, b_od, b_rd


JSON_CAGE, JSON_TET_MESH, JSON_AFFINE_BOX, JSON_AFFINE_BOX_MEMBER = range(4)


def json_roundtrip(kind: int, obj):
    """obj (a Python JSON value) -> the reference's from_json into its own class (Cage / TetMesh / AffineBoundingBox) -> its to_json -> Python value."""
    import json

    text = json.dumps(obj).encode()
    l = lib()
    l.ref_json_roundtrip.argtypes = [C.c_int, C.c_char_p, C.c_char_p, C.c_int]
    cap = 4 * len(text) + (1 << 16)
    buf = C.create_string_buffer(cap)
    n = l.ref_json_roundtrip(kind, text, buf, cap)
    assert 0 < n <= cap, n
    return json.loads(buf.value.decode())


def poisson_boundary(points, params: "abi.NsbBoundarySampling", bitfield, infer):
    """GrowingSelection::compute_poisson_boundary of the reference (its jitter is std::rand(): seed libc's generator first).
    infer(coords [n, 7]) -> [16, n] uint16 is NerfNetwork::inference_mixed_precision. Returns (density [n], shs [n, 27], coords seen by the network)."""
    pts = f32(points).reshape(-1, 3)
    n = pts.shape[0]
    bitfield = np.ascontiguousarray(bitfield, np.uint8)
    dens, shs = np.zeros(n, np.float32), np.zeros((n, 27), np.float32)
    seen = []

    def cb(_user, coords_p, m, out_p):
        coords = np.ctypeslib.as_array(coords_p, shape=(m, 7)).copy()
        seen.append(coords)
        np.ctypeslib.as_array(out_p, shape=(16, m))[:] = infer(coords)

    fn = INFER_FN(cb)
    l = lib()
    l.ref_poisson_boundary.argtypes = [C.c_void_p, C.c_uint32, C.POINTER(abi.NsbBoundarySampling), C.c_void_p, INFER_FN, C.c_void_p, C.c_void_p, C.c_void_p]
    assert l.ref_poisson_boundary(_p(pts), n, C.byref(params), _p(bitfield), fn, None, _p(dens), _p(shs)) == 0
    return dens, shs, np.concatenate(seen)


def march_trace(frame: abi.NsbFrame, bitfield, pixels, max_samples: int):
    pixels = u32(pixels)
    n = pixels.size
    bitfield = np.ascontiguousarray(bitfield, np.uint8)
    rec = np.zeros((n, max_samples, 8), np.float32)
    ray = np.zeros((n, 8), np.float32)
    cnt = np.zeros(n, np.uint32)
    alive = np.zeros(n, np.uint8)
    assert lib().ref_march_trace(C.byref(frame), _p(bitfield), _p(pixels), n, max_samples, _p(rec), _p(ray), _p(cnt), _p(alive)) == 0
    return rec, ray, cnt, alive


def _ops_array(ops):
    if not ops:
        return None, 0
    arr = (abi.NsbEditOp * len(ops))(*[o[0] for o in ops])
    return arr, len(ops)


def render(frame: abi.NsbFrame, bitfield, infer, ops=None, background=None):
    """Testbed::render_nerf of the reference. infer(coords [n, 7] float32) -> [16, n] uint16 (fp16 bits) is the network."""
    W, H = frame.width, frame.height
    bitfield = np.ascontiguousarray(bitfield, np.uint8)
    fb = np.zeros((H, W, 4), np.float32) if background is None else f32(background).copy()
    depth = np.zeros((H, W), np.float32)
    stats = np.zeros(4, np.uint64)
    batches = []

    def cb(_user, coords_p, n, out_p):
        coords = np.ctypeslib.as_array(coords_p, shape=(n, 7))
        out = infer(coords)
        batches.append(n)
        np.ctypeslib.as_array(out_p, shape=(16, n))[:] = out

    fn = INFER_FN(cb)
    arr, n_ops = _ops_array(ops)
    rc = lib().ref_render(C.byref(frame), _p(bitfield), arr, n_ops, fn, None, _p(fb), _p(depth), _p(stats))
    assert rc == 0
    return fb, depth, {"n_inferred": int(stats[1]), "n_calls": int(stats[2]), "batches": batches}


def map_rays(ops, coords):
    c = f32(coords).copy()
    mask = np.zeros(c.shape[0], np.uint8)
    arr, n_ops = _ops_array(ops)
    assert lib().ref_map_rays(arr, n_ops, _p(c), _p(mask), c.shape[0]) == 0
    return c, mask


def poisson_residuals(ops, coords):
    c = f32(coords)
    n = c.shape[0]
    sh, od, rd = np.zeros((n, 27), np.float32), np.zeros(n, np.float32), np.zeros(n, np.float32)
    arr, n_ops = _ops_array(ops)
    assert lib().ref_poisson_residuals(arr, n_ops, _p(c), n, _p(sh), _p(od), _p(rd)) == 0
    return sh, od, rd


def map_positions(ops, positions, mask):
    """EditOperator::map_positions of every operator, reverse list order. positions [n, stride] (warped position first), mask uint8 [n]."""
    p = f32(positions).copy()
    m = np.ascontiguousarray(mask, np.uint8).copy()
    arr, n_ops = _ops_array(ops)
    l = lib()
    l.ref_map_positions.argtypes = [C.POINTER(abi.NsbEditOp), C.c_int, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
    assert l.ref_map_positions(arr, n_ops, _p(p), p.shape[1], _p(m), p.shape[0]) == 0
    return p, m


def poisson_residual_density(ops, positions, density_fp16):
    """EditOperator::compute_poisson_residual_density of every operator, reverse list order: density_fp16 (uint16 bits) plus the residuals."""
    p = f32(positions).copy()
    h = np.ascontiguousarray(density_fp16).view(np.uint16).copy()
    arr, n_ops = _ops_array(ops)
    l = lib()
    l.ref_poisson_residual_density.argtypes = [C.POINTER(abi.NsbEditOp), C.c_int, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32]
    assert l.ref_poisson_residual_density(arr, n_ops, _p(p), p.shape[1], _p(h), p.shape[0]) == 0
    return h


def compute_mvc(cage_vertices, cage_tris, points, gamma=1.0, original=True):
    cv, ct, pts = f32(cage_vertices), u32(cage_tris), f32(points)
    w = np.zeros((pts.shape[0], cv.shape[0]), np.float32)
    assert lib().ref_compute_mvc(_p(cv), cv.shape[0], _p(ct), ct.shape[0], _p(pts), pts.shape[0], _p(w), gamma, int(original)) == 0
    return w


def tet_mesh_build(original_vertices, deformed_vertices, tets, amin, amax, lut_capacity=1 << 26):
    ov, dv, tt, amin, amax = f32(original_vertices), f32(deformed_vertices), u32(tets), f32(amin), f32(amax)
    n_t = tt.size // 4
    rot = np.zeros((n_t, 9), np.float32)
    off = np.zeros(abi.NSB_GRID_CELLS + 1, np.uint32)
    idx = np.zeros(lut_capacity, np.uint32)
    n_idx = C.c_uint32()
    bbox = np.zeros(12, np.float32)
    obits = np.zeros(abi.NSB_BITFIELD_BYTES, np.uint8)
    rc = lib().ref_tet_mesh_build(_p(ov), _p(dv), ov.shape[0], _p(tt), n_t, _p(amin), _p(amax), _p(rot), _p(off), _p(idx), lut_capacity, C.byref(n_idx), _p(bbox), _p(obits))
    assert rc == 0, rc
    return rot, off, idx[: n_idx.value].copy(), bbox.reshape(4, 3), obits


def svd3_rotation(A):
    A = f32(A).reshape(-1, 9)
    R = np.zeros_like(A)
    lib().ref_svd3(A.shape[0], _p(A), _p(R))
    return R


# =====================================================================================================================
# The nvcc build: the reference's own kernels and host loop on the GPU (oracle/ref_driver_cuda.cu)
# =====================================================================================================================
_culib = None


def cuda_lib() -> C.CDLL:
    global _culib
    if _culib is None:
        path = ref_build.build_cuda()
        if path is None:
            raise RuntimeError("oracle/_ref: no libnerfshop_ref_cuda.so (built where /root/reference exists; it travels with the repo)")
        l = C.CDLL(path)
        V = C.c_void_p
        l.refcu_create.restype = V
        l.refcu_create.argtypes = [V, C.POINTER(abi.NsbEditOp), C.c_int]
        l.refcu_destroy.argtypes = [V]
        l.refcu_destroy.restype = None
        l.refcu_render.argtypes = [V, C.POINTER(abi.NsbFrame), V, V, V, V, V, V]
        l.refcu_march_trace.argtypes = [V, C.POINTER(abi.NsbFrame), V, C.c_uint32, C.c_uint32, V, V, V]
        l.refcu_map_rays.argtypes = [V, V, V, C.c_uint32]
        l.refcu_poisson_residuals.argtypes = [V, V, C.c_uint32, V, V, V]
        _culib = l
    return _culib


class RefCuda:
    """A scene (occupancy bitfield + edit operators) for the reference's CUDA path. The network is `renderer`'s nsb_inference
    (NerfRenderer of this repository: the reference's tiny-cuda-nn is an absent submodule)."""

    def __init__(self, bitfield, ops=None):
        self.lib = cuda_lib()
        b = np.ascontiguousarray(bitfield, np.uint8)
        self._keep = ops
        arr, n = _ops_array(ops)
        self.h = self.lib.refcu_create(_p(b), arr, n)
        assert self.h, "refcu_create failed"

    def close(self):
        if self.h:
            self.lib.refcu_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def render(self, frame: abi.NsbFrame, renderer, fb=None, depth=None, stream: int = 0):
        """Testbed::render_nerf on the GPU into torch tensors fb [H, W, 4] / depth [H, W] (created zeroed if None)."""
        import torch

        W, H = frame.width, frame.height
        if fb is None:
            fb = torch.zeros((H, W, 4), dtype=torch.float32, device="cuda")
        if depth is None:
            depth = torch.zeros((H, W), dtype=torch.float32, device="cuda")
        fn = C.cast(renderer.lib.nsb_inference, C.c_void_p)
        stats = np.zeros(3, np.uint64)
        rc = self.lib.refcu_render(self.h, C.byref(frame), fn, renderer.ctx, fb.data_ptr(), depth.data_ptr(), stream, _p(stats))
        assert rc == 0
        return fb, depth, {"n_inferred": int(stats[0]), "n_calls": int(stats[1])}

    def march_trace(self, frame: abi.NsbFrame, pixels, max_samples: int):
        pixels = u32(pixels)
        n = pixels.size
        rec = np.zeros((n, max_samples, 8), np.float32)
        ray = np.zeros((n, 8), np.float32)
        cnt = np.zeros(n, np.uint32)
        assert self.lib.refcu_march_trace(self.h, C.byref(frame), _p(pixels), n, max_samples, _p(rec), _p(ray), _p(cnt)) == 0
        return rec, ray, cnt

    def map_rays(self, coords):
        c = f32(coords).copy()
        mask = np.zeros(c.shape[0], np.uint8)
        assert self.lib.refcu_map_rays(self.h, _p(c), _p(mask), c.shape[0]) == 0
        return c, mask

    def poisson_residuals(self, coords):
        c = f32(coords)
        n = c.shape[0]
        sh, od, rd = np.zeros((n, 27), np.float32), np.zeros(n, np.float32), np.zeros(n, np.float32)
        assert self.lib.refcu_poisson_residuals(self.h, _p(c), n, _p(sh), _p(od), _p(rd)) == 0
        return sh, od, rd
