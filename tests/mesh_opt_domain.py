"""Shared inputs of the mesh-optimisation domain tests (tests/test_mesh_opt_domain_cpu.py, tests/test_gpu_mesh_opt_domain.py).

Grid geometries, seeded models, position classes and NerfCoordinate rows come from tests/encoding_domain.py; density fields, boxes and
train AABBs from tests/mesh_domain.py. Added here:

* MESHES: meshes to optimise, each a (source, MC resolution, MC box, threshold, home train AABB) row that nsb_marching_cubes meshes on the
  device. "fox" is the synthetic scene's density on a grid of the box (its own train AABB, threshold the median raw density of the unfiltered
  points); any other source is a field of tests/mesh_domain.FIELDS or one built here. They cover the fox under a power-of-two and a
  non-power-of-two train AABB and partly outside the train AABB, many small and degenerate triangles (checkerboard), coplanar vertices
  whose cross products and normals are zero (box_zero_extent_y), coordinates near 1e6 (warped far outside the cube, 1-ring sums that lose
  precision), inf / NaN / filter values, a vertex count that is an exact multiple of 128 (no padding rows), and the fox at a resolution
  whose 2^20 and more rows take a CTA of nsb_density_gradient through several tiles.
* PARAMS: optimiser parameter rows: the reference's amounts (2048, 128, 1), each term alone, all zero, a negative amount, a threshold at a
  vertex's exact fp16 density (dens - thresh = +0 there), and thresholds of +-inf, +NaN and -NaN.
* Adam's debiasing powers: the host's powf, and powf run on the device by a small kernel built with the product's nvcc flags.
"""
from __future__ import annotations

import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

import encoding_domain as ed  # noqa: F401  (GEOMETRIES, make_model, positions, coord_rows: re-exported for the tests)
import mesh_domain as md
from nerfshop_b200 import build as nsb_build

F32 = np.float32
FOX_RES = 64
BIG_RES = 512  # the fox at this resolution has more than 2^20 vertex rows
NEG_NAN = float(np.array([0xFFC00000], np.uint32).view(F32)[0])  # quiet NaN with the sign bit set

TRAINS = {"fox": md.FOX, "non_pow2": md.TRAIN_NP, "unit": md.UNIT}


def _octahedra():
    """64 isolated inside points 2 cells apart, each the centre of an octahedron of 6 vertices: 384 = 3 x 128 vertices, no padding rows."""
    rng = np.random.default_rng(128)
    d = -rng.uniform(0.1, 1.0, (16, 16, 16)).astype(F32)
    idx = np.arange(1, 16, 4)
    for z in idx:
        for y in idx:
            for x in idx:
                d[z, y, x] = F32(rng.uniform(0.1, 1.0))
    return d, (np.array(md.BOX_NP[0], F32), np.array(md.BOX_NP[1], F32)), 0.0


# name -> (source, MC resolution (fox only), home train AABB); a non-fox source's box and threshold are its field's
MESHES = {
    "fox": ("fox", FOX_RES, "fox"),
    "fox_train_non_pow2": ("fox", FOX_RES, "non_pow2"),
    "fox_partly_outside": ("fox", FOX_RES, "unit"),
    "checkerboard": ("checkerboard", None, "non_pow2"),
    "box_zero_extent_y": ("box_zero_extent_y", None, "non_pow2"),
    "box_offset_1e6": ("box_offset_1e6", None, "fox"),
    "inf_nan_and_filter_value": ("inf_nan_and_filter_value", None, "non_pow2"),
    "octahedra_384": ("octahedra", None, "non_pow2"),
}
BIG = ("fox", BIG_RES, "fox")


def field(source):
    """(density [rz, ry, rx] float32, (box min, box max), threshold) of a non-fox source."""
    return _octahedra() if source == "octahedra" else md.FIELDS[source]


# name -> (threshold: "mesh" (the mesh's own), "vertex" (a vertex's fp16 density) or a float; smooth, density, inflate amounts)
PARAMS = {
    "reference": ("mesh", 2048.0, 128.0, 1.0),
    "smooth_only": ("mesh", 2048.0, 0.0, 0.0),
    "density_only": ("mesh", 0.0, 128.0, 0.0),
    "inflate_only": ("mesh", 0.0, 0.0, 1.0),
    "all_zero": ("mesh", 0.0, 0.0, 0.0),
    "negative_density": ("mesh", 2048.0, -128.0, 1.0),
    "thresh_at_vertex": ("vertex", 2048.0, 128.0, 1.0),
    "thresh_pos_inf": (np.inf, 2048.0, 128.0, 1.0),
    "thresh_neg_inf": (-np.inf, 2048.0, 128.0, 1.0),
    "thresh_pos_nan": (np.nan, 0.0, 128.0, 0.0),
    "thresh_neg_nan": (NEG_NAN, 0.0, 128.0, 0.0),
}


def thresh_of(kind, mesh_thresh: float, dens_u16: np.ndarray, nv: int) -> float:
    """The threshold of a PARAMS row: for "vertex", the fp16 density of the finite vertex nearest the mesh threshold."""
    if kind == "mesh":
        return float(mesh_thresh)
    if kind == "vertex":
        d = dens_u16[:nv].view(np.float16).astype(np.float64)
        ok = np.isfinite(d)
        assert ok.any()
        return float(d[ok][np.argmin(np.abs(d[ok] - mesh_thresh) if np.isfinite(mesh_thresh) else np.abs(d[ok]))])
    return float(kind)


def warp(V, train) -> np.ndarray:
    """NerfCoordinate rows of vertex rows: the position (V - mn) / (mx - mn) in float32, the one rounding warp_position makes (also for
    extents that are not powers of two); dt 0, direction 0.5."""
    mn, mx = np.array(train[0], F32), np.array(train[1], F32)
    c = np.zeros((V.shape[0], 7), F32)
    with np.errstate(invalid="ignore", over="ignore"):
        c[:, :3] = (V.astype(F32) - mn) / (mx - mn)
    c[:, 4:] = 0.5
    return c


def same_or_both_nan(a, b) -> np.ndarray:
    """Element-wise: equal bits, or both NaN (the device's NaN is canonical, the host's keeps its operand's sign and payload)."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


# ---- Adam's debiasing powers ------------------------------------------------------------------------------------------------------
def host_pows(n: int) -> np.ndarray:
    """[n, 2]: row t = the host's powf(0.9f, t), powf(0.99f, t)."""
    m = C.CDLL("libm.so.6")
    m.powf.restype, m.powf.argtypes = C.c_float, [C.c_float, C.c_float]
    return np.array([[m.powf(0.9, float(t)), m.powf(0.99, float(t))] for t in range(n)], F32)


_POW_SRC = r"""
#include <cuda_runtime.h>
#include <cstdint>
// Adam's debiasing powers as k_mesh_opt_step computes them: powf(beta, (float)t) with beta and t in registers
__global__ void k_pows(uint32_t n, float b1, float b2, float* out) {
	const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= n) return;
	out[2 * t] = powf(b1, (float)t);
	out[2 * t + 1] = powf(b2, (float)t);
}
extern "C" int device_pows(uint32_t n, float* host_out) {
	float* d = nullptr;
	if (cudaMalloc(&d, 2 * sizeof(float) * n) != cudaSuccess) return 1;
	k_pows<<<(n + 255) / 256, 256>>>(n, 0.9f, 0.99f, d);
	const cudaError_t e = cudaMemcpy(host_out, d, 2 * sizeof(float) * n, cudaMemcpyDeviceToHost);
	cudaFree(d);
	return e == cudaSuccess ? 0 : 2;
}
"""
_pow_lib = None


def pow_lib() -> C.CDLL:
    """The powers kernel, compiled into a temporary directory with the product's nvcc flags (-O3, no fast math, sm_90a)."""
    global _pow_lib
    if _pow_lib is None:
        tmp = tempfile.mkdtemp(prefix="nsb_pows_")
        atexit.register(shutil.rmtree, tmp, True)
        src, lib = os.path.join(tmp, "pows.cu"), os.path.join(tmp, "libpows.so")
        with open(src, "w") as fh:
            fh.write(_POW_SRC)
        ccbin = ["-ccbin", "/usr/bin/g++"] if os.path.exists("/usr/bin/g++") else []
        res = subprocess.run([nsb_build._nvcc()] + nsb_build.NVCC_FLAGS + ccbin + ["-o", lib, src], capture_output=True, text=True)
        assert res.returncode == 0, res.stdout + res.stderr
        l = C.CDLL(lib)
        l.device_pows.argtypes = [C.c_uint32, C.c_void_p]
        _pow_lib = l
    return _pow_lib


def device_pows(n: int) -> np.ndarray:
    """[n, 2]: row t = powf(0.9f, t), powf(0.99f, t) computed on the GPU."""
    out = np.zeros((n, 2), F32)
    assert pow_lib().device_pows(n, out.ctypes.data) == 0
    return out
