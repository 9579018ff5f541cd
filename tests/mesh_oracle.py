"""numpy restatement of the deterministic marching cubes (nsb_marching_cubes) and of the mesh checks the mesh tests share.

Vertices: one per grid edge whose end points straddle the threshold (inside = f > thresh), ordered by (grid point, axis x, y, z),
at p = {x + dt, y, z} * scale + offset with dt = (thresh - f0) / (f1 - f0) from the lower-index end. Positions are exact here when
scale is a power of two (the product is then exact, so the device's FMA rounds once like the separate add). Triangles: cells in
linear order, rows of the generated table in order.
"""
from __future__ import annotations

import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import gen_mc_table  # noqa: E402

TABLE = gen_mc_table.table()
# owner corner offset (dx, dy, dz) and axis of cube edges 0..11 (marching_cubes.cu:620-637)
EDGE_OWNER = [((0, 0, 0), 0), ((1, 0, 0), 1), ((0, 1, 0), 0), ((0, 0, 0), 1), ((0, 0, 1), 0), ((1, 0, 1), 1), ((0, 1, 1), 0), ((0, 0, 1), 1),
              ((0, 0, 0), 2), ((1, 0, 0), 2), ((1, 1, 0), 2), ((0, 1, 0), 2)]
CORNER = [(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)]


def marching_cubes(density: np.ndarray, aabb_min, aabb_max, thresh: float):
    """density: float32 [rz, ry, rx]. Returns (V float32 [nv, 3], F uint32 [nt, 3])."""
    d = np.asarray(density, np.float32)
    rz, ry, rx = d.shape
    thresh = np.float32(thresh)
    inside = d > thresh
    cross = np.zeros((rz, ry, rx, 3), bool)
    cross[:, :, :-1, 0] = inside[:, :, :-1] != inside[:, :, 1:]
    cross[:, :-1, :, 1] = inside[:, :-1, :] != inside[:, 1:, :]
    cross[:-1, :, :, 2] = inside[:-1, :, :] != inside[1:, :, :]
    flat = cross.reshape(-1)
    vid = (np.cumsum(flat) - 1).astype(np.int64).reshape(rz, ry, rx, 3)
    mn, mx = np.asarray(aabb_min, np.float32), np.asarray(aabb_max, np.float32)
    scale = (mx - mn) / np.array([rx, ry, rz], np.float32)
    zz, yy, xx, aa = np.nonzero(cross)  # C order = (z, y, x, axis) = (grid point, axis)
    f0 = d[zz, yy, xx]
    nb = [(zz, yy, xx + 1), (zz, yy + 1, xx), (zz + 1, yy, xx)]
    f1 = np.where(aa == 0, d[nb[0][0], nb[0][1], np.minimum(nb[0][2], rx - 1)],
                  np.where(aa == 1, d[nb[1][0], np.minimum(nb[1][1], ry - 1), nb[1][2]], d[np.minimum(nb[2][0], rz - 1), nb[2][1], nb[2][2]]))
    dt = (thresh - f0) / (f1 - f0)
    g = np.stack([xx, yy, zz], 1).astype(np.float32)
    g[np.arange(g.shape[0]), aa] = g[np.arange(g.shape[0]), aa] + dt
    V = (g * scale + mn).astype(np.float32)

    cfg = np.zeros((rz - 1, ry - 1, rx - 1), np.int64)
    for k, (cx, cy, cz) in enumerate(CORNER):
        cfg |= inside[cz:rz - 1 + cz, cy:ry - 1 + cy, cx:rx - 1 + cx].astype(np.int64) << k
    cz_, cy_, cx_ = np.nonzero((cfg > 0) & (cfg < 255))
    cells = cfg[cz_, cy_, cx_]
    tris = []
    for t in range(5):
        sel = np.array([len(TABLE[c]) > t for c in range(256)])[cells]
        tri = np.full((cells.size, 3), -1, np.int64)
        idx = np.nonzero(sel)[0]
        for j in range(3):
            e = np.array([TABLE[c][t][j] if len(TABLE[c]) > t else 0 for c in range(256)])[cells[idx]]
            own = np.array([EDGE_OWNER[k][0] for k in range(12)])[e]
            ax = np.array([EDGE_OWNER[k][1] for k in range(12)])[e]
            tri[idx, j] = vid[cz_[idx] + own[:, 2], cy_[idx] + own[:, 1], cx_[idx] + own[:, 0], ax]
        tris.append(tri)
    T = np.stack(tris, 1).reshape(-1, 3)  # (cell, slot) order
    F = T[T[:, 0] >= 0].astype(np.uint32)
    return V, F


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
