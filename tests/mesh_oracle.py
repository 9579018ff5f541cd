"""numpy restatement of mesh extraction on the device (nsb_density_on_grid, nsb_marching_cubes, nsb_mesh_shade) and of the mesh checks
the mesh tests share.

Vertices: one per grid edge whose end points straddle the threshold (inside = f > thresh), ordered by (grid point, axis x, y, z),
at p = fma({x + dt, y, z}, scale, offset) with dt = (thresh - f0) / (f1 - f0) from the lower-index end: the arithmetic nvcc makes of
gen_vertices' `{x + dt, y, z}.cwiseProduct(scale) + offset`, exact for every box and every field, inf and NaN included. Triangles: cells
in linear order, rows of the generated table in order.

Normals (k_mesh_normals): per vertex, the sum in ascending triangle order of (pb - pa) x (pa - pc), each cross product in its FMA form.
Colour inputs (k_mesh_colors): the network coordinate {warp(p), 0, warp(normalize(p - 0.5))}. Grid points and the filter
(k_density_on_grid): p = fma(x * (1/res), max - min, min), and the raw density is replaced by -10000 where the running density grid,
read at unwarp(warp(p)) in the cascade mip_from_pos picks, is below 0.01f.

The fp32 primitives (a correctly rounded fma, Eigen's dot product and cross product as nvcc contracts them, mip_from_pos and
cascaded_grid_idx_at) are tests/edit_domain.py's.
"""
from __future__ import annotations

import os
import sys

import numpy as np

from edit_domain import cell_index, cross3, dot3, fma, mip_from_pos

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gen_mc_table  # noqa: E402

F32 = np.float32
TABLE = gen_mc_table.table()
# owner corner offset (dx, dy, dz) and axis of cube edges 0..11 (marching_cubes.cu:620-637)
EDGE_OWNER = [((0, 0, 0), 0), ((1, 0, 0), 1), ((0, 1, 0), 0), ((0, 0, 0), 1), ((0, 0, 1), 0), ((1, 0, 1), 1), ((0, 1, 1), 0), ((0, 0, 1), 1),
              ((0, 0, 0), 2), ((1, 0, 0), 2), ((1, 1, 0), 2), ((0, 1, 0), 2)]
CORNER = [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)]
GRID_CELLS = 128 ** 3
MIN_OPTICAL_THICKNESS = F32(0.01)
FILTERED = F32(-10000.0)


def cell_configs(density: np.ndarray, thresh: float) -> np.ndarray:
    """The configuration (bit k: corner k inside) of every cell of a float32 [rz, ry, rx] field."""
    d = np.asarray(density, F32)
    rz, ry, rx = d.shape
    inside = d > F32(thresh)
    cfg = np.zeros((rz - 1, ry - 1, rx - 1), np.int64)
    for k, (cx, cy, cz) in enumerate(CORNER):
        cfg |= inside[cz:rz - 1 + cz, cy:ry - 1 + cy, cx:rx - 1 + cx].astype(np.int64) << k
    return cfg


def marching_cubes(density: np.ndarray, aabb_min, aabb_max, thresh: float):
    """density: float32 [rz, ry, rx]. Returns (V float32 [nv, 3], F uint32 [nt, 3])."""
    d = np.asarray(density, F32)
    rz, ry, rx = d.shape
    thresh = F32(thresh)
    inside = d > thresh
    cross = np.zeros((rz, ry, rx, 3), bool)
    cross[:, :, :-1, 0] = inside[:, :, :-1] != inside[:, :, 1:]
    cross[:, :-1, :, 1] = inside[:, :-1, :] != inside[:, 1:, :]
    cross[:-1, :, :, 2] = inside[:-1, :, :] != inside[1:, :, :]
    flat = cross.reshape(-1)
    vid = (np.cumsum(flat) - 1).astype(np.int64).reshape(rz, ry, rx, 3)
    mn, mx = np.asarray(aabb_min, F32), np.asarray(aabb_max, F32)
    with np.errstate(all="ignore"):  # inf and NaN densities, thresholds and extents go through as the device computes them
        scale = (mx - mn) / np.array([rx, ry, rz], F32)
        zz, yy, xx, aa = np.nonzero(cross)  # C order = (z, y, x, axis) = (grid point, axis)
        f0 = d[zz, yy, xx]
        nb = [(zz, yy, xx + 1), (zz, yy + 1, xx), (zz + 1, yy, xx)]
        f1 = np.where(aa == 0, d[nb[0][0], nb[0][1], np.minimum(nb[0][2], rx - 1)],
                      np.where(aa == 1, d[nb[1][0], np.minimum(nb[1][1], ry - 1), nb[1][2]], d[np.minimum(nb[2][0], rz - 1), nb[2][1], nb[2][2]]))
        dt = (thresh - f0) / (f1 - f0)
        g = np.stack([xx, yy, zz], 1).astype(F32)
        g[np.arange(g.shape[0]), aa] = g[np.arange(g.shape[0]), aa] + dt
        V = fma(g, scale[None, :], mn[None, :]).reshape(-1, 3)

    cfg = cell_configs(d, thresh)
    cz_, cy_, cx_ = np.nonzero((cfg > 0) & (cfg < 255))
    cells = cfg[cz_, cy_, cx_]
    tris = []
    for t in range(5):
        sel = np.array([len(TABLE[c]) > t for c in range(256)])[cells]
        tri = np.full((cells.size, 3), -1, np.int64)
        idx = np.nonzero(sel)[0]
        for j in range(3):
            e = np.array([TABLE[c][t][j] if len(TABLE[c]) > t else 0 for c in range(256)])[cells[idx]]
            own = np.array([EDGE_OWNER[k][0] for k in range(12)], np.int64).reshape(12, 3)[e]
            ax = np.array([EDGE_OWNER[k][1] for k in range(12)])[e]
            tri[idx, j] = vid[cz_[idx] + own[:, 2], cy_[idx] + own[:, 1], cx_[idx] + own[:, 0], ax]
        tris.append(tri)
    T = np.stack(tris, 1).reshape(-1, 3)  # (cell, slot) order
    F = T[T[:, 0] >= 0].astype(np.uint32)
    return V, F


def padded_rows(nv: int) -> int:
    """The vertex rows the mesh arrays have: n_vertices rounded up to 128 (marching_cubes.cu:751)."""
    return (int(nv) + 127) // 128 * 128


def normals(V, F, nv: int, rows: int) -> np.ndarray:
    """k_mesh_normals: rows [rows, 3]; vertex v < nv gets the float32 sum, in ascending triangle order, of (pb - pa) x (pa - pc) over
    its triangles; the padding rows are zero."""
    V = np.asarray(V, F32)
    F = np.asarray(F, np.int64).reshape(-1, 3)
    out = np.zeros((rows, 3), F32)
    with np.errstate(all="ignore"):
        pa, pb, pc = V[F[:, 0]], V[F[:, 1]], V[F[:, 2]]
        tn = cross3(pb - pa, pa - pc)
        # one incidence per (triangle, corner) in triangle order: np.add.at adds them one at a time, so each vertex sums in that order
        np.add.at(out, F.reshape(-1), np.repeat(tn, 3, axis=0))
    out[nv:] = 0
    return out


def _normalized(d):
    """Eigen's normalized(): d / sqrt(dot(d, d)) when dot(d, d) > 0, d unchanged otherwise (dot in its FMA form)."""
    n2 = dot3(d, d)
    nn = np.sqrt(np.where(n2 > 0, n2, F32(1.0))).astype(F32)
    return np.where((n2 > 0)[:, None], d / nn[:, None], d).astype(F32)


def warp_position(p, mn, mx):
    return ((np.asarray(p, F32) - mn) / (mx - mn)).astype(F32)


def unwarp_position(pw, mn, mx):
    return fma(pw, (mx - mn)[None, :], mn[None, :])


def color_inputs(V, train_aabb) -> np.ndarray:
    """generate_nerf_network_inputs_from_positions as k_mesh_colors computes it: NerfCoordinate rows [n, 7] = {warp_position(p), warp_dt
    of the minimum step (0), warp_direction(normalize(p - 0.5))}."""
    V = np.asarray(V, F32).reshape(-1, 3)
    mn, mx = np.asarray(train_aabb[0], F32), np.asarray(train_aabb[1], F32)
    out = np.zeros((V.shape[0], 7), F32)
    with np.errstate(all="ignore"):
        d = _normalized((V - F32(0.5)).astype(F32))
        out[:, :3] = warp_position(V, mn, mx)
        out[:, 4:] = ((d + F32(1.0)) * F32(0.5)).astype(F32)
    return out


def grid_positions(res, render_aabb, train_aabb, rows=None):
    """k_density_on_grid's grid points (generate_grid_samples_nerf_uniform), x fastest: (world positions p [n, 3], warped positions
    [n, 3]); only the given point indices when rows is given."""
    r = np.asarray(res, np.int64)
    i = np.arange(int(np.prod(r)), dtype=np.int64) if rows is None else np.asarray(rows, np.int64)
    xyz = np.stack([i % r[0], (i // r[0]) % r[1], i // (r[0] * r[1])], 1).astype(F32)
    rmn, rmx = np.asarray(render_aabb[0], F32), np.asarray(render_aabb[1], F32)
    tmn, tmx = np.asarray(train_aabb[0], F32), np.asarray(train_aabb[1], F32)
    inv = (F32(1.0) / r.astype(F32)).astype(F32)
    p = fma((xyz * inv).astype(F32), (rmx - rmn)[None, :], rmn[None, :])
    return p, warp_position(p, tmn, tmx)


def filtered(pw, train_aabb, density_grid) -> np.ndarray:
    """grid_samples_half_to_float's filter at warped positions pw: the density grid (float [5 * 128^3]) at unwarp(pw), in the cascade
    mip_from_pos gives, is below NERF_MIN_OPTICAL_THICKNESS."""
    tmn, tmx = np.asarray(train_aabb[0], F32), np.asarray(train_aabb[1], F32)
    p = unwarp_position(pw, tmn, tmx)
    mip = mip_from_pos(p)
    cell = cell_index(p, mip).astype(np.int64) + mip.astype(np.int64) * GRID_CELLS
    return np.asarray(density_grid, F32)[cell] < MIN_OPTICAL_THICKNESS


def half_to_float(pw, raw_u16, train_aabb, density_grid=None) -> np.ndarray:
    """grid_samples_half_to_float: the raw fp16 density as float, -10000 where the filter applies (no filter without a grid)."""
    v = np.asarray(raw_u16, np.uint16).view(np.float16).astype(F32)
    if density_grid is None:
        return v
    return np.where(filtered(pw, train_aabb, density_grid), FILTERED, v)


def edge_manifold(F: np.ndarray) -> bool:
    """Every undirected edge is used by exactly two triangles, once in each direction."""
    F = np.asarray(F, np.int64)
    e = np.concatenate([F[:, [0, 1]], F[:, [1, 2]], F[:, [2, 0]]])
    key = np.unique(e[:, 0] * (1 << 32) + e[:, 1], return_counts=True)
    if (key[1] != 1).any():
        return False  # a directed edge used twice
    und = np.unique(np.minimum(e[:, 0], e[:, 1]) * (1 << 32) + np.maximum(e[:, 0], e[:, 1]), return_counts=True)
    return bool((und[1] == 2).all())


def euler_characteristic(F: np.ndarray) -> int:
    F = np.asarray(F, np.int64)
    e = np.concatenate([F[:, [0, 1]], F[:, [1, 2]], F[:, [2, 0]]])
    n_e = np.unique(np.minimum(e[:, 0], e[:, 1]) * (1 << 32) + np.maximum(e[:, 0], e[:, 1])).size
    return int(np.unique(F).size - n_e + F.shape[0])


def boundary_cycles(tris):
    """The directed boundary cycles of one cell's triangles (edges used once and not in reverse), each rotated to its smallest edge."""
    de = {}
    for a, b, c in tris:
        for u, v in ((a, b), (b, c), (c, a)):
            de[(u, v)] = de.get((u, v), 0) + 1
    nxt = {u: v for (u, v), n in de.items() if (v, u) not in de}
    out = set()
    seen = set()
    for s in nxt:
        if s in seen:
            continue
        cyc, e = [], s
        while e not in seen:
            seen.add(e)
            cyc.append(e)
            e = nxt[e]
        k = cyc.index(min(cyc))
        out.add(tuple(cyc[k:] + cyc[:k]))
    return frozenset(out)


# ---- comparisons ----------------------------------------------------------------------------------------------------------------
def bits(a) -> np.ndarray:
    """The uint32 bits of a float32 array with every NaN made the same NaN: bit-for-bit comparisons that count all NaNs as equal."""
    a = np.array(a, F32, copy=True)
    a[np.isnan(a)] = np.float32(np.nan)
    return a.view(np.uint32)


def vertex_multiset(V) -> np.ndarray:
    """The rows of V as sorted (x, y, z) bit triples (NaNs equal)."""
    b = np.ascontiguousarray(bits(np.asarray(V, F32).reshape(-1, 3)))
    return np.sort(b.view([("x", "<u4"), ("y", "<u4"), ("z", "<u4")]).reshape(-1))


def cell_cycle_edges(V, F) -> np.ndarray:
    """The directed edges that remain of all triangles once every edge used in both directions cancels, keyed by the end points'
    position bits (NaNs equal): rows (u bits 3, v bits 3, net count) in sorted order. Inside one cell the diagonals of a triangulation
    cancel, so what remains is the sum of every cell's boundary cycles with their direction, whichever way each cycle is triangulated:
    the reference's table triangulates some cycles differently from tools/gen_mc_table.py's, whose cycles it shares."""
    F = np.asarray(F, np.int64).reshape(-1, 3)
    b = bits(np.asarray(V, F32).reshape(-1, 3))
    e = np.concatenate([F[:, [0, 1]], F[:, [1, 2]], F[:, [2, 0]]])
    u, v = b[e[:, 0]], b[e[:, 1]]
    uv = np.concatenate([u, v], 1)
    vu = np.concatenate([v, u], 1)
    # orient each edge from its lexicographically smaller end point: +1 along, -1 against
    less = np.zeros(len(e), np.int64)
    for k in range(3):
        undecided = less == 0
        less[undecided & (u[:, k] < v[:, k])] = 1
        less[undecided & (u[:, k] > v[:, k])] = -1
    key = np.where((less >= 0)[:, None], uv, vu)
    if key.shape[0] == 0:
        return np.zeros((0, 7), np.int64)
    uniq, inv = np.unique(key, axis=0, return_inverse=True)
    net = np.zeros(uniq.shape[0], np.int64)
    np.add.at(net, inv.reshape(-1), less)
    keep = net != 0
    return np.concatenate([uniq[keep].astype(np.int64), net[keep, None]], 1)
