"""Shared inputs of the encoding-domain tests: a table of hash-grid geometries, a seeded model for any of them, position classes
inside and outside the unit cube, and the host build of the product's grid index (nsb_device.cuh compiled by nvcc for the CPU)."""
from __future__ import annotations

import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

import numpy as np

from nerfshop_b200 import abi, synthetic as syn

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(REPO, "nerfshop_b200", "csrc")


def desc(log2: int = 19, base: int = 16, pls: float | None = None, aabb_scale: int = 4) -> abi.NsbModelDesc:
    if pls is None:
        pls = syn.per_level_scale(aabb_scale, 16, base)
    return abi.NsbModelDesc(16, 2, log2, base, pls, 64, 1, 2, 4)


# name -> description; what each row exercises is in the comment
GEOMETRIES = {
    "fox": desc(aabb_scale=4),                         # levels 0-3 dense: an all-dense pair and all-hashed pairs
    "aabb1": desc(aabb_scale=1),                       # mixed pair (4, 5)
    "aabb2": desc(aabb_scale=2),
    "aabb16": desc(aabb_scale=16),
    "aabb128": desc(aabb_scale=128),                   # level 15: res 2^18, tcnn's uint32 stride wraps to 0 and the level is indexed densely
    "log2_12": desc(log2=12, aabb_scale=4),            # level 0 res^3 = 4096 = 2^12 (dense/hashed tie), mixed pair (0, 1)
    "log2_3": desc(log2=3, aabb_scale=4),              # every level hashed, 8 entries
    "base1_pls2": desc(base=1, pls=2.0),               # scale 0 at level 0 (res 1)
    "log2_22": desc(log2=22, aabb_scale=4),            # large tables, dense levels up to res 161
    "log2_24_aabb128": desc(log2=24, aabb_scale=128),
}


def level_geometry(d: abi.NsbModelDesc):
    """(scale, res, size, hashed) per level, tcnn's rule for hashed (uint32 stride, may wrap)."""
    scale, res, _, size, _ = syn.level_table(d)
    hashed = []
    for l in range(d.n_levels):
        stride, dim = 1, 0
        while dim < 3 and stride <= int(size[l]):
            stride = (stride * int(res[l])) & 0xFFFFFFFF
            dim += 1
        hashed.append(int(size[l]) < stride)
    return scale, res, size, np.array(hashed)


def make_model(d: abi.NsbModelDesc, seed: int) -> np.ndarray:
    """Seeded fp16 parameter block for any description: Xavier-uniform MLP weights, then noise tables in [-0.5, 0.5)."""
    rng = np.random.default_rng(seed)
    _, _, _, _, entries = syn.level_table(d)
    mats = [(64, 32), (16, 64), (64, 32), (64, 64), (16, 64)]
    parts = [rng.uniform(-1, 1, o * i) * np.sqrt(6.0 / (o + i)) for o, i in mats]
    parts.append(rng.uniform(-0.5, 0.5, 2 * int(entries)))
    return np.concatenate(parts).astype(np.float16).view(np.uint16)


def positions(scale: np.ndarray, res: np.ndarray, size: np.ndarray, hashed: np.ndarray, seed: int = 0, n_random: int = 64) -> np.ndarray:
    """Per-axis values of every position class; rows combine them so each axis sees every class."""
    rng = np.random.default_rng(seed)
    v = [rng.random(n_random).astype(np.float32)]
    v.append(np.array([0.0, 1.0, np.nextafter(np.float32(1), np.float32(2))], np.float32))
    for l in range(len(scale)):
        if not hashed[l] and scale[l] > 0:
            e = np.float32(-0.5) / scale[l]
            v.append(np.array([e, np.nextafter(e, np.float32(-1)), np.nextafter(e, np.float32(1))], np.float32))
            v.append((np.arange(0, int(res[l]), max(1, int(res[l]) // 4)) / scale[l]).astype(np.float32))  # lattice points
    v.append(np.array([-0.04, -0.3, 1.3, -2.0, 3.5, 1e3, -1e3, 1e6, -1e6], np.float32))
    return np.unique(np.concatenate(v))


SPECIALS = np.array([np.inf, -np.inf, np.nan], np.float32)


def coord_rows(axis_values: np.ndarray, seed: int = 1, specials: bool = True) -> np.ndarray:
    """NerfCoordinate rows (n x 7): every axis value on each axis against random partners, plus the specials."""
    rng = np.random.default_rng(seed)
    vals = np.concatenate([axis_values, SPECIALS]) if specials else axis_values
    rows = []
    for a in range(3):
        p = rng.choice(vals, size=(vals.size, 3)).astype(np.float32)
        p[:, a] = vals
        rows.append(p)
    p = np.concatenate(rows)
    out = np.zeros((p.shape[0], 7), np.float32)
    out[:, :3] = p
    out[:, 3] = 0.01
    out[:, 4:] = rng.random((p.shape[0], 3)).astype(np.float32)
    return out


def grid_coords(f: np.ndarray, scale: float) -> np.ndarray:
    """The grid coordinate of a position on one level as the device computes it: cvt.rzi.s32.f32(floor(fma(scale, x, 0.5)))."""
    with np.errstate(invalid="ignore", over="ignore"):
        p = (np.float64(scale) * f.astype(np.float64) + 0.5).astype(np.float32)  # fma: exact product + add, one rounding
    g = np.floor(p).astype(np.float64)
    g = np.where(np.isnan(g), 0.0, np.clip(g, -2.0 ** 31, 2.0 ** 31 - 1))
    return g.astype(np.int64).astype(np.uint32)


# ---- host build of the product's grid index ----
_HELPER = r"""
#include "nsb_device.cuh"
using namespace nsb;
extern "C" int host_levels(const NsbModelDesc* d, uint32_t* res, uint32_t* size, uint32_t* hashed, uint64_t* n_entries, int* in_range) {
	DevLevel L[MAX_LEVELS];
	if (!build_levels(d, L, n_entries)) return 1;
	for (uint32_t l = 0; l < d->n_levels; ++l) { res[l] = L[l].res; size[l] = L[l].size; hashed[l] = L[l].hashed; }
	*in_range = dense_in_range(L, d->n_levels) ? 1 : 0;
	return 0;
}
extern "C" int host_grid_index(const NsbModelDesc* d, uint32_t level, int mode, int in_range, const uint32_t* g, uint32_t n, uint32_t* out) {
	DevLevel L[MAX_LEVELS];
	uint64_t e;
	if (!build_levels(d, L, &e) || level >= d->n_levels) return 1;
	const DevLevel& V = L[level];
	for (uint32_t i = 0; i < n; ++i) {
		const uint32_t x = g[3 * i], y = g[3 * i + 1], z = g[3 * i + 2];
		if (in_range) out[i] = mode == 0 ? grid_index<0, true>(V, x, y, z) : mode == 1 ? grid_index<1, true>(V, x, y, z) : grid_index<2, true>(V, x, y, z);
		else out[i] = mode == 0 ? grid_index<0>(V, x, y, z) : mode == 1 ? grid_index<1>(V, x, y, z) : grid_index<2>(V, x, y, z);
	}
	return 0;
}
"""

_host_lib = None


def host_lib() -> C.CDLL:
    """nsb_device.cuh's build_levels and grid_index, compiled by nvcc for the host into a temporary directory."""
    global _host_lib
    if _host_lib is None:
        nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
        tmp = tempfile.mkdtemp(prefix="nsb_grid_index_")
        atexit.register(shutil.rmtree, tmp, True)  # the loaded library stays mapped until exit; the directory goes with it
        src, lib = os.path.join(tmp, "helper.cu"), os.path.join(tmp, "libhelper.so")
        with open(src, "w") as fh:
            fh.write(_HELPER)
        ccbin = ["-ccbin", "/usr/bin/g++"] if os.path.exists("/usr/bin/g++") else []
        cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared", *ccbin, "-I", CSRC, "-o", lib, src]
        res = subprocess.run(cmd, capture_output=True, text=True)
        assert res.returncode == 0, res.stdout + res.stderr
        l = C.CDLL(lib)
        l.host_levels.argtypes = [C.POINTER(abi.NsbModelDesc)] + [C.c_void_p] * 5
        l.host_grid_index.argtypes = [C.POINTER(abi.NsbModelDesc), C.c_uint32, C.c_int, C.c_int, C.c_void_p, C.c_uint32, C.c_void_p]
        _host_lib = l
    return _host_lib
