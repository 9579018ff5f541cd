"""The mesh-extraction input domain, shared by tests/test_mesh_domain_cpu.py and tests/test_gpu_mesh_domain.py.

Fields (FIELDS): density grids for marching cubes, built directly (no network), each with the box it is meshed over and its threshold:
seeded random fields that together reach all 254 non-trivial cell configurations; quantised fields where many values equal the threshold
(dt = 0 or 1, coincident vertices, zero-area triangles); a checkerboard (4 triangles in every cell); a sphere cut by the grid's faces;
infinities, NaN, the filter value -10000, +-3e38 (f1 - f0 overflows), subnormals about a threshold of 0, +-0 against thresholds +0 and
-0; thresholds of +-inf, NaN and +-FLT_MAX; grids wholly inside and wholly outside (empty meshes); boxes that are not powers of two,
inverted on one axis, of zero extent on one axis, and offset by about 1e6; and a grid of 516 tiles of 1024 points whose crossings lie
in tiles 511, 512 and 515, on both sides of the 512-tile chunks of the tile scan.

Each field is small enough that the reference's whole result fits one stored file (tests/ref_golden.py) without row sampling.

Grid queries (QUERIES): render boxes (a power of two, not a power of two, partly and wholly outside the train AABB, inverted, and one
whose grid points land on the cascade boundaries |p - 0.5| = 2^k and on the AABB centre) over the fox-config train AABB, the unit cube
and a non-cubic train AABB that is not a power of two, at resolutions (16,16,16), (48,16,16), (16,32,80) and (128,128,128). Density
grids (density_grids()): the synthetic scene's occupancy as 0/1, and a seeded float grid made of 0.01f, its two float neighbours, 0, -0,
negatives, NaN, +inf and values well above the filter.
"""
from __future__ import annotations

import numpy as np

import mesh_oracle as mo

F32 = np.float32
FLT_MAX = float(np.finfo(F32).max)

FOX = ((-1.5, -1.5, -1.5), (2.5, 2.5, 2.5))
UNIT = ((0.0, 0.0, 0.0), (1.0, 1.0, 1.0))
TRAIN_NP = ((-1.1, -0.7, -1.3), (2.3, 1.9, 2.1))  # non-cubic, no extent a power of two
BOX_NP = ((-1.3, -1.1, -0.9), (2.2, 2.1, 2.4))


def _signs(rng, shape):
    return np.where(rng.random(shape) < 0.5, F32(-1.0), F32(1.0)).astype(F32)


def _sprinkle(rng, d, values, share):
    """d with a share of its points replaced by values drawn from `values`."""
    d = d.copy()
    m = rng.random(d.shape) < share
    d[m] = rng.choice(np.asarray(values, F32), size=int(m.sum()))
    return d


def _sphere(shape, centre, radius):
    rz, ry, rx = shape
    z, y, x = np.meshgrid(np.arange(rz), np.arange(ry), np.arange(rx), indexing="ij")
    return (F32(radius) - np.sqrt((x - centre[0]) ** 2 + (y - centre[1]) ** 2 + (z - centre[2]) ** 2)).astype(F32)


def _long_grid():
    """16 x 16 x 2064 points (516 tiles): -1 everywhere but for single inside points in tiles 0, 511, 512 and 515 (one tile = 4 z slices)."""
    d = np.full((16 * 129, 16, 16), -1.0, F32)
    for tile, (x, y, dz) in ((0, (3, 4, 1)), (511, (7, 8, 2)), (512, (5, 9, 0)), (512, (12, 2, 3)), (515, (9, 10, 1))):
        d[4 * tile + dz, y, x] = 1.0
    return d


def _fields():
    f = {}
    rng = np.random.default_rng(20261018)
    # seeded random fields: +-1 (dt = 1/2 everywhere) and random magnitudes
    f["random_pm1"] = (_signs(rng, (16, 16, 16)), BOX_NP, 0.0)
    f["random_magnitudes"] = ((_signs(rng, (16, 16, 16)) * rng.uniform(0.01, 1.0, (16, 16, 16))).astype(F32), FOX, 0.0)
    f["random_pm1_b"] = (_signs(rng, (16, 16, 16)), TRAIN_NP, 0.0)
    # many values equal to the threshold
    f["quantised"] = (rng.choice(np.array([-1.0, -0.5, 0.0, 0.5, 1.0], F32), (16, 16, 16)), BOX_NP, 0.0)
    f["quantised_at_threshold"] = (rng.choice(np.array([0.0, 0.25, 0.25, 0.5], F32), (16, 16, 16)), FOX, 0.25)
    z, y, x = np.meshgrid(np.arange(16), np.arange(16), np.arange(16), indexing="ij")
    f["checkerboard"] = (np.where((x + y + z) % 2 == 0, F32(1.0), F32(-1.0)).astype(F32), BOX_NP, 0.0)
    f["sphere_cut_by_faces"] = (_sphere((16, 32, 48), (40.5, 10.25, 3.0), 11.0), BOX_NP, 0.0)
    # special values
    base = (_signs(rng, (16, 16, 16)) * rng.uniform(0.01, 1.0, (16, 16, 16))).astype(F32)
    f["inf_nan_and_filter_value"] = (_sprinkle(rng, base, [np.inf, -np.inf, np.nan, -10000.0], 0.15), BOX_NP, 0.0)
    f["overflowing_differences"] = ((_signs(rng, (16, 16, 16)) * rng.choice(np.array([3e38, FLT_MAX, 1.0], F32), (16, 16, 16))).astype(F32), FOX, 0.0)
    sub = np.array([-3, -2, -1, 1, 2, 3], np.int32)
    f["subnormals_about_zero"] = (np.ldexp(rng.choice(sub, (16, 16, 16)).astype(F32), -149).astype(F32), BOX_NP, 0.0)
    f["subnormals_about_subnormal"] = (np.ldexp(rng.integers(0, 9, (16, 16, 16)).astype(F32), -149).astype(F32), FOX, float(np.ldexp(F32(4), -149)))
    zeros = rng.choice(np.array([0.0, -0.0, 1.0, -1.0], F32), (16, 16, 16))
    f["signed_zeros_thresh_pos0"] = (zeros, BOX_NP, 0.0)
    f["signed_zeros_thresh_neg0"] = (zeros, BOX_NP, -0.0)
    specials = _sprinkle(rng, base, [np.inf, -np.inf, np.nan, FLT_MAX, -FLT_MAX], 0.2)
    f["thresh_pos_inf"] = (specials, BOX_NP, np.inf)
    f["thresh_neg_inf"] = (specials, BOX_NP, -np.inf)
    f["thresh_nan"] = (specials, BOX_NP, np.nan)
    f["thresh_flt_max"] = (specials, BOX_NP, FLT_MAX)
    f["thresh_neg_flt_max"] = (specials, BOX_NP, -FLT_MAX)
    f["all_inside"] = (np.full((16, 16, 16), 1.0, F32), BOX_NP, 0.0)
    f["all_outside"] = (np.full((16, 16, 16), -1.0, F32), BOX_NP, 0.0)
    # boxes
    sphere = _sphere((16, 16, 16), (7.3, 8.1, 6.6), 5.2)
    f["box_inverted_x"] = (sphere, ((2.2, -1.1, -0.9), (-1.3, 2.1, 2.4)), 0.0)
    f["box_zero_extent_y"] = (sphere, ((-1.3, 0.7, -0.9), (2.2, 0.7, 2.4)), 0.0)
    f["box_offset_1e6"] = (sphere, ((1.0e6 + 0.3, -1.0e6 - 0.7, 1.0e6), (1.0e6 + 3.9, -1.0e6 + 2.6, 1.0e6 + 3.3)), 0.0)
    f["long_grid_tile_chunks"] = (_long_grid(), BOX_NP, 0.0)
    return {k: (np.ascontiguousarray(d, F32), (np.array(b[0], F32), np.array(b[1], F32)), float(t)) for k, (d, b, t) in f.items()}


FIELDS = _fields()
RANDOM_FIELDS = ("random_pm1", "random_magnitudes", "random_pm1_b")
EMPTY_FIELDS = ("thresh_pos_inf", "thresh_nan", "all_inside", "all_outside")  # no point is inside, or every point is


def res_of(name):
    """(rx, ry, rz) of a field: its array is [rz, ry, rx]."""
    rz, ry, rx = FIELDS[name][0].shape
    return np.array([rx, ry, rz], np.int32)


def config_coverage():
    """The non-trivial cell configurations (1..254) the random fields reach together."""
    seen = set()
    for k in RANDOM_FIELDS:
        d, _, t = FIELDS[k]
        seen |= set(np.unique(mo.cell_configs(d, t)).tolist())
    return seen - {0, 255}


# ---- grid queries ---------------------------------------------------------------------------------------------------------------
BOXES = {
    "pow2": FOX,
    "non_pow2": BOX_NP,
    "partly_outside": ((-2.7, -0.4, 1.1), (1.3, 3.9, 4.6)),
    "wholly_outside": ((2.75, -3.5, -3.2), (5.6, -1.6, -1.7)),
    "inverted": ((2.2, -1.1, 2.4), (-1.3, 2.1, -0.9)),
    "cascade_boundaries": ((-3.5, -3.5, -3.5), (4.5, 4.5, 4.5)),  # at res 16 and 32, p - 0.5 = k / 2 or k / 4: 0 and +-2^k included
}
TRAINS = {"fox": FOX, "unit": UNIT, "non_pow2": TRAIN_NP}
QUERIES = {
    "pow2_fox_16": ((16, 16, 16), "pow2", "fox"),
    "pow2_fox_128": ((128, 128, 128), "pow2", "fox"),
    "pow2_unit_128": ((128, 128, 128), "pow2", "unit"),
    "non_pow2_fox_48": ((48, 16, 16), "non_pow2", "fox"),
    "non_pow2_non_pow2_16_32_80": ((16, 32, 80), "non_pow2", "non_pow2"),
    "non_pow2_unit_48": ((48, 16, 16), "non_pow2", "unit"),
    "partly_outside_fox_16_32_80": ((16, 32, 80), "partly_outside", "fox"),
    "partly_outside_non_pow2_48": ((48, 16, 16), "partly_outside", "non_pow2"),
    "wholly_outside_fox_16": ((16, 16, 16), "wholly_outside", "fox"),
    "inverted_fox_48": ((48, 16, 16), "inverted", "fox"),
    "cascade_boundaries_fox_16": ((16, 16, 16), "cascade_boundaries", "fox"),
    "cascade_boundaries_non_pow2_32": ((32, 32, 32), "cascade_boundaries", "non_pow2"),
    "cascade_boundaries_unit_16": ((16, 16, 16), "cascade_boundaries", "unit"),
}
MAX_ROWS = 12288  # grid points compared with the reference per query: all of them up to this count, else the first and last 4096 and a seeded rest


def query(name):
    """(res int32 [3], render AABB (min, max), train AABB (min, max)) as float32 arrays."""
    res, box, train = QUERIES[name]
    b, t = BOXES[box], TRAINS[train]
    return np.array(res, np.int32), (np.array(b[0], F32), np.array(b[1], F32)), (np.array(t[0], F32), np.array(t[1], F32))


def query_rows(res, seed=0, k=MAX_ROWS):
    """Sorted grid-point indices: all points when there are at most k, else the first and last 4096 and a seeded sample between."""
    n = int(np.prod(np.asarray(res, np.int64)))
    if n <= k:
        return np.arange(n, dtype=np.int64)
    rng = np.random.default_rng(seed + n)
    mid = rng.choice(np.arange(4096, n - 4096), size=k - 8192, replace=False)
    return np.sort(np.concatenate([np.arange(4096), mid, np.arange(n - 4096, n)])).astype(np.int64)


def float_density_grid(seed=5):
    """A running density grid (float [5 * 128^3]) of filter edge values: 0.01f and its neighbours, +-0, negatives, NaN, +inf, 0.5."""
    t = F32(0.01)
    vals = np.array([t, np.nextafter(t, F32(0)), np.nextafter(t, F32(1)), 0.0, -0.0, -1.0, -0.01, np.nan, np.inf, 0.5], F32)
    return np.random.default_rng(seed).choice(vals, 5 * 128 ** 3).astype(F32)


def density_grids(occ):
    return {"occupancy": np.unpackbits(occ, bitorder="little").astype(F32), "float": float_density_grid()}
