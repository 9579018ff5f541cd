"""TetMesh::vanish (tet_mesh.cu:251-363) restated on the host, the meshes both vanish tests run it on, and the reference's own vanish.

The cells vanish clears are the cells build_tet_grid's cell test marks: nsb_build_tet_grid's `bitfield` output ("set where a tet
touches the cell", pinned to the reference's build_tet_grid by tests/test_oracle_vs_ref.py). Vanishing on the host is therefore: zero
the density and clear the occupancy bit wherever that bitfield is set.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from nerfshop_b200 import abi, editing

N_CELLS, N_BYTES = abi.NSB_GRID_CELLS, abi.NSB_BITFIELD_BYTES


def touched_bitfield(vertices, tets):
    """The cells (bit cell % 8 of byte cell / 8, cell = level * 128^3 + morton) that tets over `vertices` touch, at every cascade."""
    lib = abi.load_library()
    v, t = np.ascontiguousarray(vertices, np.float32).reshape(-1, 3), np.ascontiguousarray(tets, np.uint32).reshape(-1, 4)
    off = np.zeros(N_CELLS + 1, np.uint32)
    bits = np.zeros(N_BYTES, np.uint8)
    n = C.c_uint64()
    st = lib.nsb_build_tet_grid(v.ctypes.data, v.shape[0], t.ctypes.data, t.shape[0], off.ctypes.data, None, 0, C.byref(n), bits.ctypes.data)
    assert st == 0, st
    return bits


def touched_cells(vertices, tets):
    return np.unpackbits(touched_bitfield(vertices, tets), bitorder="little").astype(bool)


def host_vanish(grid, bitfield, vertices, tets):
    """(grid, bitfield) after vanish; grid may be None (then only the bitfield is cleared)."""
    touched = touched_bitfield(vertices, tets)
    g = None
    if grid is not None:
        g = np.array(grid, np.float32, copy=True)
        g[np.unpackbits(touched, bitorder="little").astype(bool)] = 0.0
    return g, np.asarray(bitfield, np.uint8) & ~touched


def inputs(seed=0):
    """A running grid with every kind of value vanish may meet (positive, zero, negative zero, negative) and a patterned bitfield."""
    rng = np.random.default_rng(seed)
    grid = rng.uniform(0.0, 2.0, N_CELLS).astype(np.float32)
    grid[::5] = 0.0
    grid[1::7] = -0.0
    grid[2::11] = -1.0
    bits = np.full(N_BYTES, 0xFF, np.uint8)
    bits[::3] = 0x5A
    bits[1::13] = 0x00
    return grid, bits


def meshes(model):
    """name -> (original vertices, deformed vertices, tets): the shapes vanish has to handle."""
    out = {}
    c = editing.lattice_cage(model, (0.5, 0.62, 0.78), (0.17, 0.17, 0.17), n_lattice=4)  # the tet-grid pin's cage
    out["lattice4"] = (c.original_vertices, c.vertices, c.tets)
    c = editing.lattice_cage(model, (0.41, 0.30, 0.33), (0.08, 0.14, 0.08), pull=(0.05, -0.04, 0.05), n_lattice=3)
    out["pulled"] = (c.original_vertices, c.vertices, c.tets)
    # tets dozens of cascade-3 cells wide, outside cascades 0 and 1 (their boxes clamp to the grid's edge cells there)
    v, t = editing.lattice_tets((1.3, -2.9, 1.2), (3.9, -1.1, 3.6), 1)
    out["coarse"] = (v, v, t)
    # straddles the unit cube's and the train aabb's +x and -z faces
    amax, amin = np.asarray(model.aabb_max, np.float32), np.asarray(model.aabb_min, np.float32)
    v, t = editing.lattice_tets((0.93, 0.4, -0.06), (amax[0] + 0.07, 0.55, 0.08), 3)
    v2, t2 = editing.lattice_tets((amin[0] - 0.05, 0.2, amin[2] - 0.05), (amin[0] + 0.05, 0.3, amin[2] + 0.05), 2)
    out["boundary"] = (np.concatenate([v, v2]), np.concatenate([v, v2]), np.concatenate([t, t2 + v.shape[0]]))
    # one zero-volume tet: four coplanar vertices
    v = np.array([[0.3, 0.4, 0.5], [0.6, 0.45, 0.5], [0.35, 0.7, 0.5], [0.55, 0.6, 0.5]], np.float32)
    out["flat"] = (v, v, np.array([[0, 1, 2, 3]], np.uint32))
    return out


def reference_vanish(original_vertices, vertices, tets, amin, amax, grid, bitfield):
    """The reference's own TetMesh::vanish (oracle/_ref/libnerfshop_ref_vanish.so) on copies of grid / bitfield. Returned losslessly and
    small enough to store: (packed mask of the grid entries whose bits changed, their new values, the whole new bitfield). The wall time of
    the vanish call alone is left in reference_vanish.seconds."""
    from oracle import ref_vanish_build

    lib = C.CDLL(ref_vanish_build.build())
    V = C.c_void_p
    lib.ref_tet_mesh_vanish.argtypes = [V, V, C.c_uint32, V, C.c_uint32, V, V, V, V, C.POINTER(C.c_double)]
    ov, dv = np.ascontiguousarray(original_vertices, np.float32), np.ascontiguousarray(vertices, np.float32)
    tt = np.ascontiguousarray(tets, np.uint32)
    amin, amax = np.ascontiguousarray(amin, np.float32), np.ascontiguousarray(amax, np.float32)
    g, b = np.array(grid, np.float32, copy=True), np.array(bitfield, np.uint8, copy=True)
    secs = C.c_double()
    rc = lib.ref_tet_mesh_vanish(ov.ctypes.data, dv.ctypes.data, ov.shape[0], tt.ctypes.data, tt.size // 4, amin.ctypes.data, amax.ctypes.data,
                                 g.ctypes.data, b.ctypes.data, C.byref(secs))
    assert rc == 0, rc
    reference_vanish.seconds = secs.value
    changed = g.view(np.uint32) != np.asarray(grid, np.float32).view(np.uint32)
    return np.packbits(changed, bitorder="little"), g[changed], b


def apply_stored(grid, stored):
    """The reference's grid and bitfield from reference_vanish's result."""
    mask_packed, values, bits = stored
    g = np.array(grid, np.float32, copy=True)
    g[np.unpackbits(mask_packed, bitorder="little").astype(bool)] = values
    return g, bits
