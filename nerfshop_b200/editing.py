"""Host-side mirror of the reference's edit operators (include/neural-graphics-primitives/editing/):

  CageDeformation   <- CageDeformation + GrowingSelection's tet_interpolation_mesh/proxy_cage
                       (cage_deformation.{h,cu}, growing_selection.cu:1514-1660, tet_mesh.{h,cu}, cage.{h,cu})
  AffineDuplication <- AffineDuplication (affine_duplication.{h,cu})

The interactive tooling that CREATES a cage in the reference (region growing, marching cubes, decimation, TetGen)
is out of scope (SURVEY.md §2 row 11); here a cage is given as vertices + triangles and the tet mesh as a
Kuhn-subdivided lattice of the cage's bounding box. Everything geometric runs in the C library's host code
(nsb_compute_mvc / nsb_interpolate_with_mvc / nsb_local_rotations / nsb_build_tet_grid).
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import abi


def _fptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _uptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint32))


def box_cage(bmin, bmax):
    """8 vertices + 12 outward CCW triangles of an axis-aligned box (GUI default cage, testbed.cu:1118-1150)."""
    bmin, bmax = np.asarray(bmin, np.float32), np.asarray(bmax, np.float32)
    v = np.array([[x, y, z] for x in (bmin[0], bmax[0]) for y in (bmin[1], bmax[1]) for z in (bmin[2], bmax[2])], np.float32)
    # vertex id = 4*ix + 2*iy + iz
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    tris = []
    for a, b, c, d in quads:
        tris += [(a, b, c), (a, c, d)]
    return v, np.array(tris, np.uint32)


def lattice_tets(bmin, bmax, n: int):
    """(n+1)^3 lattice vertices and 6 n^3 Kuhn tetrahedra (a conforming mesh without TetGen)."""
    bmin, bmax = np.asarray(bmin, np.float64), np.asarray(bmax, np.float64)
    g = np.linspace(0.0, 1.0, n + 1)
    Z, Y, X = np.meshgrid(g, g, g, indexing="ij")
    verts = (bmin + np.stack([X, Y, Z], -1).reshape(-1, 3) * (bmax - bmin)).astype(np.float32)

    def vid(i, j, k):
        return i + (n + 1) * (j + (n + 1) * k)

    perms = [(0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)]
    tets = []
    for k in range(n):
        for j in range(n):
            for i in range(n):
                for p in perms:
                    c = [i, j, k]
                    ids = [vid(*c)]
                    for ax in p:
                        c[ax] += 1
                        ids.append(vid(*c))
                    tets.append(ids)
    return verts, np.array(tets, np.uint32)


class CageDeformation:
    def __init__(self, scene_aabb_min, scene_aabb_max, cage_vertices, cage_triangles, tet_vertices, tets, copy=False, local_rotations=True):
        self.lib = abi.load_library()
        self.aabb_min = np.asarray(scene_aabb_min, np.float32)
        self.aabb_max = np.asarray(scene_aabb_max, np.float32)
        self.cage_original = np.ascontiguousarray(cage_vertices, np.float32)
        self.cage_vertices = self.cage_original.copy()
        self.cage_triangles = np.ascontiguousarray(cage_triangles, np.uint32).reshape(-1, 3)
        self.original_vertices = np.ascontiguousarray(tet_vertices, np.float32)
        self.vertices = self.original_vertices.copy()
        self.tets = np.ascontiguousarray(tets, np.uint32).reshape(-1, 4)
        self.copy = bool(copy)
        self.use_local_rotations = bool(local_rotations)
        self.apply_poisson = False
        self.residual_amplitude = 1.0
        self.boundary_shs = None
        self.boundary_outside_density = None
        self.boundary_residual_density = None
        # GrowingSelection::initialize_mvc (growing_selection.cu:1599): weights w.r.t. the ORIGINAL cage
        nv, nc = self.original_vertices.shape[0], self.cage_original.shape[0]
        self.mvc = np.zeros((nv, nc), np.float32)
        st = self.lib.nsb_compute_mvc(self.cage_original.ctypes.data, nc, self.cage_triangles.ctypes.data, self.cage_triangles.shape[0],
                                      self.original_vertices.ctypes.data, nv, 0.0, self.mvc.ctypes.data)
        assert st == 0
        self.original_bitfield = np.zeros(abi.NSB_BITFIELD_BYTES, np.uint8)
        off = np.zeros(abi.NSB_GRID_CELLS + 1, np.uint32)
        n = C.c_uint64()
        self._grid(self.original_vertices, off, self.original_bitfield)  # build_original_tet_grid: canonical occupancy
        self.update_tet_mesh()

    @classmethod
    def from_arrays(cls, scene_aabb_min, scene_aabb_max, cage_original, cage_vertices, cage_triangles, tet_original_vertices, tets, mvc,
                    gamma_coordinates=None, copy=False, local_rotations=True):
        """An operator restored from saved arrays (GrowingSelection(json) + TetMesh(json), growing_selection.cu:81-117): the MVC
        weights are taken as stored, the deformed vertices / rotations / lookup table are rebuilt (build_tet_grid, :114)."""
        self = cls.__new__(cls)
        self.lib = abi.load_library()
        self.aabb_min, self.aabb_max = np.asarray(scene_aabb_min, np.float32), np.asarray(scene_aabb_max, np.float32)
        self.cage_original = np.ascontiguousarray(cage_original, np.float32).reshape(-1, 3)
        self.cage_vertices = np.ascontiguousarray(cage_vertices, np.float32).reshape(-1, 3)
        self.cage_triangles = np.ascontiguousarray(cage_triangles, np.uint32).reshape(-1, 3)
        self.original_vertices = np.ascontiguousarray(tet_original_vertices, np.float32).reshape(-1, 3)
        self.vertices = self.original_vertices.copy()
        self.tets = np.ascontiguousarray(tets, np.uint32).reshape(-1, 4)
        self.copy, self.use_local_rotations = bool(copy), bool(local_rotations)
        self.apply_poisson, self.residual_amplitude = False, 1.0
        self.boundary_shs = self.boundary_outside_density = self.boundary_residual_density = None
        self.mvc = np.ascontiguousarray(mvc, np.float32).reshape(self.original_vertices.shape[0], self.cage_original.shape[0])
        self.gamma_coordinates = self.mvc if gamma_coordinates is None else np.ascontiguousarray(gamma_coordinates, np.float32).reshape(self.mvc.shape)
        self.original_bitfield = np.zeros(abi.NSB_BITFIELD_BYTES, np.uint8)
        self._grid(self.original_vertices, np.zeros(abi.NSB_GRID_CELLS + 1, np.uint32), self.original_bitfield)
        self.update_tet_mesh()
        return self

    def _grid(self, verts, offsets, bitfield):
        n = C.c_uint64()
        st = self.lib.nsb_build_tet_grid(verts.ctypes.data, verts.shape[0], self.tets.ctypes.data, self.tets.shape[0], offsets.ctypes.data, None, 0,
                                         C.byref(n), None if bitfield is None else bitfield.ctypes.data)
        assert st == 0, st
        idx = np.zeros(max(int(n.value), 1), np.uint32)
        st = self.lib.nsb_build_tet_grid(verts.ctypes.data, verts.shape[0], self.tets.ctypes.data, self.tets.shape[0], offsets.ctypes.data, idx.ctypes.data,
                                         idx.size, C.byref(n), None if bitfield is None else bitfield.ctypes.data)
        assert st == 0, st
        return idx[: int(n.value)]

    def set_membrane(self, shs, outside_density, residual_density, amplitude=1.0, apply=True):
        """TetMesh::boundary_*_gpu arrays (tet_mesh.h:91-94), one entry per tet-mesh vertex."""
        nv = self.vertices.shape[0]
        self.boundary_shs = np.ascontiguousarray(shs, np.float32).reshape(nv, 27)
        self.boundary_outside_density = np.ascontiguousarray(outside_density, np.float32).reshape(nv)
        self.boundary_residual_density = np.ascontiguousarray(residual_density, np.float32).reshape(nv)
        self.residual_amplitude = float(amplitude)
        self.apply_poisson = bool(apply)

    def update_tet_mesh(self):
        """GrowingSelection::update_tet_mesh (growing_selection.cu:1615): MVC -> bboxes -> rotations -> LUT."""
        nv, nc = self.vertices.shape[0], self.cage_vertices.shape[0]
        st = self.lib.nsb_interpolate_with_mvc(self.mvc.ctypes.data, nv, nc, self.cage_vertices.ctypes.data, self.vertices.ctypes.data)
        assert st == 0
        self.rotations = np.zeros((self.tets.shape[0], 9), np.float32)
        st = self.lib.nsb_local_rotations(self.vertices.ctypes.data, self.original_vertices.ctypes.data, self.tets.ctypes.data, self.tets.shape[0], self.rotations.ctypes.data)
        assert st == 0
        self.lut_offsets = np.zeros(abi.NSB_GRID_CELLS + 1, np.uint32)
        self.lut_idx = self._grid(self.vertices, self.lut_offsets, None)

    def _warp(self, p):
        return ((np.asarray(p, np.float32) - self.aabb_min) / (self.aabb_max - self.aabb_min)).astype(np.float32)

    def to_op(self):
        """(NsbEditOp, keepalive): the POD of interpolate_tet's arguments (cage_deformation.cu:558-573)."""
        op = abi.NsbEditOp()
        op.type = abi.NSB_OP_CAGE
        op.copy = int(self.copy)
        op.apply_poisson = int(self.apply_poisson)
        op.residual_amplitude = self.residual_amplitude
        bmin, bmax = self.vertices.min(0), self.vertices.max(0)            # TetMesh::post_update_vertices (tet_mesh.cu:13-20)
        obmin, obmax = self.original_vertices.min(0), self.original_vertices.max(0)
        for i in range(3):
            op.scene_aabb_min[i], op.scene_aabb_max[i] = float(self.aabb_min[i]), float(self.aabb_max[i])
            op.bbox_min[i], op.bbox_max[i] = float(bmin[i]), float(bmax[i])
        wmin, wmax, owmin, owmax = self._warp(bmin), self._warp(bmax), self._warp(obmin), self._warp(obmax)
        for i in range(3):
            op.warped_bbox_min[i], op.warped_bbox_max[i] = float(wmin[i]), float(wmax[i])
            op.original_warped_bbox_min[i], op.original_warped_bbox_max[i] = float(owmin[i]), float(owmax[i])
        op.n_tets, op.n_vertices, op.n_lut_idx = self.tets.shape[0], self.vertices.shape[0], self.lut_idx.size
        keep = dict(
            off=self.lut_offsets, idx=np.ascontiguousarray(self.lut_idx), tets=np.ascontiguousarray(self.tets.reshape(-1)),
            v=np.ascontiguousarray(self.vertices.reshape(-1)), ov=np.ascontiguousarray(self.original_vertices.reshape(-1)),
            rot=np.ascontiguousarray(self.rotations.reshape(-1)), bits=self.original_bitfield,
        )
        op.tet_lut_offsets = _uptr(keep["off"])
        op.tet_lut_idx = _uptr(keep["idx"])
        op.tets = _uptr(keep["tets"])
        op.vertices = _fptr(keep["v"])
        op.original_vertices = _fptr(keep["ov"])
        if self.use_local_rotations:
            op.local_rotations = _fptr(keep["rot"])
        op.original_bitfield = keep["bits"].ctypes.data_as(C.POINTER(C.c_uint8))
        # each membrane array may be absent on its own (NULL)
        for name, field, arr in (("shs", "boundary_shs", self.boundary_shs), ("od", "boundary_outside_density", self.boundary_outside_density),
                                 ("rd", "boundary_residual_density", self.boundary_residual_density)):
            if arr is not None:
                keep[name] = np.ascontiguousarray(arr, np.float32).reshape(-1)
                setattr(op, field, _fptr(keep[name]))
        return op, keep


def affine_box(center, scale, rot=None):
    """AffineBoundingBox (affine_bounding_box.cuh): min, u, v, w, center of an oriented box."""
    R = np.eye(3, dtype=np.float32) if rot is None else np.asarray(rot, np.float32)
    center, scale = np.asarray(center, np.float32), np.asarray(scale, np.float32)
    b = abi.NsbAffineBox()
    mn = (-0.5 * (R @ scale) + center).astype(np.float32)
    u, v, w = R @ (scale[0] * np.array([1, 0, 0], np.float32)), R @ (scale[1] * np.array([0, 1, 0], np.float32)), R @ (scale[2] * np.array([0, 0, 1], np.float32))
    for i in range(3):
        b.min[i], b.u[i], b.v[i], b.w[i], b.center[i] = float(mn[i]), float(u[i]), float(v[i]), float(w[i]), float(center[i])
    return b


class AffineDuplication:
    """Copy/move a box of space. All quantities are in WARPED coordinates like the reference's m_warped_* members."""

    def __init__(self, sel_center_w, sel_scale_w, translation_w, scale=(1, 1, 1), rotation=None, hide_original=True, correct_dir=False):
        self.R = np.eye(3, dtype=np.float32) if rotation is None else np.asarray(rotation, np.float32)
        self.sel_center = np.asarray(sel_center_w, np.float32)
        self.sel_scale = np.asarray(sel_scale_w, np.float32)
        self.translation = np.asarray(translation_w, np.float32)
        self.scale = np.asarray(scale, np.float32)
        self.hide_original = hide_original
        self.correct_dir = correct_dir

    def to_op(self):
        op = abi.NsbEditOp()
        op.type = abi.NSB_OP_AFFINE
        op.selection_box = affine_box(self.sel_center, self.sel_scale)
        op.destination_box = affine_box(self.sel_center + self.translation, self.sel_scale * self.scale, self.R)
        for i in range(3):
            op.translation[i] = float(self.translation[i])
            op.scale[i] = float(self.scale[i])
        flat = self.R.T.reshape(-1)  # column-major
        for i in range(9):
            op.rotation[i] = float(flat[i])
        op.hide_original = int(self.hide_original)
        op.correct_dir = int(self.correct_dir)
        return op, {}


def lattice_cage(model, center, half, pull=(0.10, 0.03, 0.0), n_lattice=3, copy=False, membrane_seed=None):
    """A box cage around `center` (world units) with a lattice tet mesh inside it (5-6 tets per lattice cube; TetGen is not available),
    its +x face pulled by `pull`; optionally seeded membrane (Poisson) arrays. Used by the test fixtures (E1 / E3 of SURVEY.md section 8d) and by
    bench.py's edit configurations."""
    center, half = np.asarray(center, np.float32), np.asarray(half, np.float32)
    cv, ct = box_cage(center - half, center + half)
    tv, tets = lattice_tets(center - 0.97 * half, center + 0.97 * half, n_lattice)
    op = CageDeformation(model.aabb_min, model.aabb_max, cv, ct, tv, tets, copy=copy)
    moved = op.cage_original.copy()
    moved[moved[:, 0] > center[0]] += np.asarray(pull, np.float32)  # pull the +x face
    op.cage_vertices = moved
    op.update_tet_mesh()
    if membrane_seed is not None:
        rng = np.random.default_rng(membrane_seed)
        nv = op.vertices.shape[0]
        shs = rng.uniform(-0.3, 0.3, (nv, 27)).astype(np.float32)
        shs[:, [0, 9, 18]] += 1.2  # DC terms: a visible base colour
        op.set_membrane(shs, rng.uniform(0.0, 30.0, nv).astype(np.float32), rng.uniform(-2.0, 6.0, nv).astype(np.float32), amplitude=1.0, apply=True)
    return op
