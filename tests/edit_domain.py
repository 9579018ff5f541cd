"""The edit operators' input domain, shared by tests/test_edit_domain_cpu.py and tests/test_gpu_edit_domain.py.

Operator sets (SETS): lists of edit objects (editing.CageDeformation, editing.AffineDuplication, EmptyOp) that build the cases random
fixtures never do: cages across cascade boundaries and the train AABB's faces, inverted and flattened tets, overlapping operators in both
list orders, copy cages, affine duplications in every flag combination, cages without rotations, operators without tets, and membranes
with every subset of their three arrays.

Sample sets (samples()): warped NerfCoordinate rows on the places where the operators branch: tet-mesh vertices, edge midpoints and face
points (rest and deformed meshes; a face point of the rest mesh lies exactly on a shared face), lookup-table cell faces, cascade
boundaries, the warped boxes' faces, affine-box faces, and random points in and around each operator; every point with its ulp
neighbours on both sides.

The cages are built on dyadic coordinates (centre, half size and lattice spacing are short binary fractions) so that rest-mesh points and
their warped coordinates are exact, and a point on a shared face is on it in fp32 too.

map_rays_lut_free() restates EditOperator::map_rays without the lookup table (interpolate_tet, cage_deformation.cu:197-269;
point_in_tet / bary_tet, selection_utils.h:10-47; translate_in_box, affine_duplication.cu:92-118): every tet is tested and the
lowest-index containing tet wins, which is the first entry of the sample's cell list, whose entries are in ascending tet order.
"""
from __future__ import annotations

import numpy as np

from nerfshop_b200 import editing

F32, F64 = np.float32, np.float64


# ---- fp32 arithmetic as the device contracts it ------------------------------------------------------------------------------
def fma(a, b, c):
    """fmaf, correctly rounded: the fp32 product is exact in float64, TwoSum gives the sum's rounding error, and a sum that the float64
    rounding left exactly halfway between two floats is nudged towards the error before the one rounding to fp32 (without the nudge,
    the dyadic coordinates of the domain hit the double-rounding case in a few samples per ten thousand)."""
    p = np.asarray(a, F32).astype(F64) * np.asarray(b, F32).astype(F64)
    c = np.asarray(c, F32).astype(F64)
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)
    with np.errstate(invalid="ignore"):
        s = np.where(err != 0, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(F32)


def dot3(a, b):   # Eigen's reduction tree x0*y0 + (x1*y1 + x2*y2) as nvcc contracts it: fma(x,x', fma(y,y', z*z'))
    return fma(a[..., 0], b[..., 0], fma(a[..., 1], b[..., 1], (a[..., 2] * b[..., 2]).astype(F32)))


def cross3(a, b):  # fma(a.y, b.z, -(a.z*b.y)), ...
    return np.stack([fma(a[..., 1], b[..., 2], -(a[..., 2] * b[..., 1]).astype(F32)), fma(a[..., 2], b[..., 0], -(a[..., 0] * b[..., 2]).astype(F32)),
                     fma(a[..., 0], b[..., 1], -(a[..., 1] * b[..., 0]).astype(F32))], -1)


def same_side(v1, v2, v3, v4, p):
    n = cross3(v2 - v1, v3 - v1)
    return np.signbit(dot3(n, v4 - v1)) == np.signbit(dot3(n, p - v1))


def stp(a, b, c):
    return dot3(a, cross3(b, c))


def mip_from_pos(p):
    m = np.abs(p - F32(0.5)).max(-1)
    return np.clip(np.frexp(m)[1] + 1, 0, 4)


def _expand_bits(v):
    v = v.astype(np.uint32)
    v = (v * np.uint32(0x00010001)) & np.uint32(0xFF0000FF)
    v = (v * np.uint32(0x00000101)) & np.uint32(0x0F00F00F)
    v = (v * np.uint32(0x00000011)) & np.uint32(0xC30C30C3)
    v = (v * np.uint32(0x00000005)) & np.uint32(0x49249249)
    return v


def cell_index(p, level):
    """cascaded_grid_idx_at (common_nerf.cu:117-136) of finite positions p [n, 3] at levels [n]."""
    s = np.ldexp(F32(1.0), -level.astype(np.int32)).astype(F32)[:, None]
    q = fma(p - F32(0.5), s, F32(0.5))
    i = np.clip(np.trunc((q * F32(128.0)).astype(F32)), 0, 127).astype(np.uint32)
    return _expand_bits(i[:, 0]) | (_expand_bits(i[:, 1]) << np.uint32(1)) | (_expand_bits(i[:, 2]) << np.uint32(2))


def _v(a):
    return np.array(a[:], F32)


# ---- operators -----------------------------------------------------------------------------------------------------------------
class EmptyOp:
    """A cage operator whose tet mesh is empty (n_tets == 0): every entry point skips it, whatever its boxes say."""

    def __init__(self, cage):
        self.cage = cage

    def to_op(self):
        op, keep = self.cage.to_op()
        op.n_tets = op.n_vertices = op.n_lut_idx = 0
        for f in ("tet_lut_offsets", "tet_lut_idx", "tets", "vertices", "original_vertices", "local_rotations", "original_bitfield",
                  "boundary_shs", "boundary_outside_density", "boundary_residual_density"):
            setattr(op, f, None)
        return op, keep


def dyadic_cage(model, center, half, pull=(0.0625, 0.03125, 0.0), n=4, copy=False, rotations=True):
    """A box cage centre +- half (world units, short binary fractions) around a Kuhn lattice of n^3 cubes on centre +- 7/8 half, its
    +x face pulled by `pull`. The cage weights are the trilinear ones (generalised barycentric coordinates of a box, stored like saved MVC
    weights): dyadic, so the deformed vertices are exact too, and a dyadic combination of a tet's vertices lies exactly on its face in fp32."""
    center, half = np.asarray(center, F64), np.asarray(half, F64)
    cv, ct = editing.box_cage(center - half, center + half)   # vertex id 4*ix + 2*iy + iz
    tv, tets = editing.lattice_tets(center - 0.875 * half, center + 0.875 * half, n)
    u = (tv.astype(F64) - (center - half)) / (2 * half)
    w = np.stack([np.prod([u[:, a] if (j >> (2 - a)) & 1 else 1 - u[:, a] for a in range(3)], 0) for j in range(8)], 1).astype(F32)
    moved = cv.copy()
    moved[moved[:, 0] > center[0]] += np.asarray(pull, F32)
    op = editing.CageDeformation.from_arrays(model.aabb_min, model.aabb_max, cv, moved, ct, tv, tets, w, copy=copy, local_rotations=rotations)
    assert np.array_equal(op.vertices, (w.astype(F64) @ moved.astype(F64)).astype(F32)), "deformed vertices must be exact"
    return op


def flattened_cage(model, center, half):
    """One lattice cube (6 Kuhn tets) whose vertices follow the cage corners exactly (one-hot MVC weights), dragged so that corner (1,0,0)
    lands on the midpoint of the (0,0,0)-(1,1,0) diagonal: the tet (000, 100, 110, 111) becomes flat, with zero volume in fp32."""
    center, half = np.asarray(center, F64), np.asarray(half, F64)
    cv, ct = editing.box_cage(center - half, center + half)   # vertex id 4*ix + 2*iy + iz
    tv, tets = editing.lattice_tets(center - half, center + half, 1)  # vertex id ix + 2*iy + 4*iz
    mvc = np.zeros((8, 8), F32)
    for v in range(8):
        ix, iy, iz = v & 1, (v >> 1) & 1, v >> 2
        mvc[v, 4 * ix + 2 * iy + iz] = 1.0
    moved = cv.copy()
    moved[4] = (cv[0] + cv[6]) / 2  # corner (1,0,0) -> midpoint of corners (0,0,0), (1,1,0)
    return editing.CageDeformation.from_arrays(model.aabb_min, model.aabb_max, cv, moved, ct, tv, tets, mvc)


def with_membrane(op, seed, arrays=("shs", "od", "rd"), amplitude=1.0, apply=True):
    """Seeded membrane arrays; `arrays` names the ones the operator keeps (the others stay NULL)."""
    rng = np.random.default_rng(seed)
    nv = op.vertices.shape[0]
    shs = rng.uniform(-0.3, 0.3, (nv, 27)).astype(F32)
    shs[:, [0, 9, 18]] += 1.2
    op.set_membrane(shs, rng.uniform(0.0, 30.0, nv).astype(F32), rng.uniform(-2.0, 6.0, nv).astype(F32), amplitude=amplitude, apply=apply)
    for name, attr in (("shs", "boundary_shs"), ("od", "boundary_outside_density"), ("rd", "boundary_residual_density")):
        if name not in arrays:
            setattr(op, attr, None)
    return op


_ROT = np.array([[0.8, -0.6, 0.0], [0.6, 0.8, 0.0], [0.0, 0.0, 1.0]], F32)
_ROT_X = np.array([[1.0, 0.0, 0.0], [0.0, 0.6, -0.8], [0.0, 0.8, 0.6]], F32)


def _to_warped(model, p):
    return ((np.asarray(p, F32) - model.aabb_min) / (model.aabb_max - model.aabb_min)).astype(F32)


def _affine(model, center_world, half_world, shift_world, **kw):
    """AffineDuplication of the box centre +- half (world units), moved by shift; all three given in warped units as the reference keeps them."""
    diag = model.aabb_max - model.aabb_min
    return editing.AffineDuplication(_to_warped(model, center_world), (2 * np.asarray(half_world, F32) / diag).astype(F32),
                                     (np.asarray(shift_world, F32) / diag).astype(F32), **kw)


def _partial(model, arrays):
    return [with_membrane(dyadic_cage(model, (0.5, 0.625, 0.75), (0.125, 0.125, 0.125)), 11, amplitude=0.75),
            with_membrane(dyadic_cage(model, (0.5625, 0.625, 0.75), (0.125, 0.125, 0.125), pull=(0.0, 0.0625, 0.0)), 12, arrays=arrays, amplitude=1.5)]


def _sets():
    head = dict(center=(0.5, 0.625, 0.75), half=(0.125, 0.125, 0.125))
    s = {
        # a tet that crosses a cascade boundary is listed at both levels: x = 1 (cascade 0/1), x = 1.5 (1/2)
        "cascade_0_1": lambda m: [dyadic_cage(m, (1.0, 0.625, 0.5), (0.125, 0.125, 0.125))],
        "cascade_1_2": lambda m: [dyadic_cage(m, (1.5, 0.5, -0.5), (0.1875, 0.125, 0.1875), pull=(0.0625, 0.0, 0.03125))],
        # the train AABB is [-1.5, 2.5]^3: warped coordinates leave [0, 1]
        "train_aabb_faces": lambda m: [dyadic_cage(m, (2.5, 2.5, 0.5), (0.125, 0.125, 0.125), pull=(0.0625, -0.03125, 0.0))],
        # the +x face dragged past the -x face: every tet inverted (negative volume)
        "inverted": lambda m: [dyadic_cage(m, **head, pull=(-0.375, 0.0, 0.0))],
        "flattened": lambda m: [flattened_cage(m, (0.5, 0.625, 0.75), (0.125, 0.125, 0.125))],
        "overlap_moves_ab": lambda m: [dyadic_cage(m, **head), dyadic_cage(m, (0.625, 0.625, 0.75), (0.125, 0.125, 0.125), pull=(0.0, 0.0625, 0.03125))],
        "overlap_moves_ba": lambda m: [dyadic_cage(m, (0.625, 0.625, 0.75), (0.125, 0.125, 0.125), pull=(0.0, 0.0625, 0.03125)), dyadic_cage(m, **head)],
        "copy_under_move": lambda m: [dyadic_cage(m, **head, copy=True), dyadic_cage(m, (0.5625, 0.6875, 0.75), (0.125, 0.125, 0.125), pull=(0.0, 0.0, 0.0625))],
        "cage_then_affine": lambda m: [dyadic_cage(m, **head), _affine(m, (0.5, 0.625, 0.75), (0.1, 0.1, 0.1), (0.125, 0.0625, 0.0), rotation=_ROT)],
        "affine_then_cage": lambda m: [_affine(m, (0.5, 0.625, 0.75), (0.1, 0.1, 0.1), (0.125, 0.0625, 0.0), rotation=_ROT), dyadic_cage(m, **head)],
        "no_rotations": lambda m: [dyadic_cage(m, **head, rotations=False)],
        "no_tets": lambda m: [dyadic_cage(m, (0.5625, 0.625, 0.75), (0.125, 0.125, 0.125)), EmptyOp(dyadic_cage(m, **head, pull=(0.25, 0.0, 0.0)))],
        "membranes_overlap": lambda m: [with_membrane(dyadic_cage(m, **head), 5, amplitude=0.5),
                                        with_membrane(dyadic_cage(m, (0.5625, 0.625, 0.75), (0.125, 0.125, 0.125), pull=(0.0, 0.0625, 0.0)), 6, amplitude=2.5)],
        "membrane_not_applied": lambda m: [with_membrane(dyadic_cage(m, **head), 7, apply=False)],
    }
    for hide in (False, True):
        for cdir in (False, True):
            s[f"affine_hide{int(hide)}_dir{int(cdir)}"] = (lambda hide, cdir: lambda m: [
                _affine(m, (0.5, 0.5, 0.5), (0.125, 0.125, 0.125), (0.1875, 0.0625, -0.125), scale=(1.25, 0.75, 1.0), rotation=_ROT_X,
                        hide_original=hide, correct_dir=cdir)])(hide, cdir)
    for arrays in (("shs",), ("od",), ("rd",), ("shs", "od"), ("shs", "rd"), ("od", "rd")):
        s["membrane_" + "_".join(arrays)] = (lambda a: lambda m: _partial(m, a))(arrays)
    return s


SETS = _sets()
NAMES = sorted(SETS)


def build(model, name):
    return SETS[name](model)


def ops_of(items):
    return [it.to_op() for it in items]


def cages_of(items):
    return [it for it in items if isinstance(it, editing.CageDeformation)]


# ---- samples -------------------------------------------------------------------------------------------------------------------
def _mesh_points(verts, tets):
    """Vertices, edge midpoints, face centroids and dyadic face points (a + b + 2c) / 4, in float64."""
    v = verts.astype(F64)
    T = tets.astype(np.int64)
    edges = np.unique(np.sort(np.concatenate([T[:, [i, j]] for i in range(4) for j in range(i + 1, 4)]), axis=1), axis=0)
    faces = np.unique(np.sort(np.concatenate([T[:, [0, 1, 2]], T[:, [0, 1, 3]], T[:, [0, 2, 3]], T[:, [1, 2, 3]]]), axis=1), axis=0)
    fa, fb, fc = v[faces[:, 0]], v[faces[:, 1]], v[faces[:, 2]]
    return np.concatenate([v, (v[edges[:, 0]] + v[edges[:, 1]]) / 2, (fa + fb + fc) / 3, (fa + fb + 2 * fc) / 4, (2 * fa + fb + fc) / 4])


def _ulp_neighbours(w):
    w = w.astype(F32)
    return np.concatenate([w, np.nextafter(w, F32(-np.inf)), np.nextafter(w, F32(np.inf))])


def _on_planes(rng, lo, hi, axis_values, n_per):
    """Points in the box [lo, hi] (warped) with one coordinate set to each of axis_values[a] in turn."""
    out = []
    for a in range(3):
        for val in axis_values[a]:
            p = (lo + rng.random((n_per, 3)) * (hi - lo)).astype(F32)
            p[:, a] = val
            out.append(p)
    return np.concatenate(out) if out else np.zeros((0, 3), F32)


def _world_planes(model, lo_w, hi_w, planes):
    """Warped coordinates of the world planes (e.g. cascade boundaries) that cross the world box [lo_w, hi_w], per axis."""
    return [[_to_warped(model, np.full(3, x, F32))[a] for x in planes if lo_w[a] <= x <= hi_w[a]] for a in range(3)]


def samples(model, items, seed=0, n_random=3000):
    """Warped NerfCoordinate rows [n, 7] (position, dt, direction) on the branch points of `items`, with ulp neighbours."""
    rng = np.random.default_rng(seed)
    diag = (model.aabb_max - model.aabb_min).astype(F64)
    pts = []
    for it in items:
        if isinstance(it, EmptyOp):
            it = it.cage
        if isinstance(it, editing.CageDeformation):
            for verts in (it.original_vertices, it.vertices):
                pts.append(_to_warped(model, _mesh_points(verts, it.tets)))
            op, _ = it.to_op()
            boxes = [(_v(op.warped_bbox_min), _v(op.warped_bbox_max)), (_v(op.original_warped_bbox_min), _v(op.original_warped_bbox_max))]
            for lo, hi in boxes:
                pts.append(_on_planes(rng, lo, hi, [[lo[a], hi[a]] for a in range(3)], 40))
            lo = np.minimum(boxes[0][0], boxes[1][0])
            hi = np.maximum(boxes[0][1], boxes[1][1])
        else:
            op, _ = it.to_op()
            lo, hi = np.full(3, np.inf, F32), np.full(3, -np.inf, F32)
            for b in (op.selection_box, op.destination_box):
                mn, u, v, w = _v(b.min), _v(b.u), _v(b.v), _v(b.w)
                # du == 0 is inside, du == |u|^2 outside: points on each face, half-open side included
                a, c = rng.random((60, 1)).astype(F32), rng.random((60, 1)).astype(F32)
                for e, f, g in ((u, v, w), (v, w, u), (w, u, v)):
                    pts.append((mn + a * f + c * g).astype(F32))
                    pts.append((mn + e + a * f + c * g).astype(F32))
                corners = np.array([mn + i * u + j * v + k * w for i in (0, 1) for j in (0, 1) for k in (0, 1)], F32)
                lo, hi = np.minimum(lo, corners.min(0)), np.maximum(hi, corners.max(0))
        # lookup-table cell faces: world p with (p - 0.5) * 2^-level + 0.5 a multiple of 1/128, levels 0-2, inside the operator's box
        lo_w, hi_w = (lo.astype(F64) * diag + model.aabb_min), (hi.astype(F64) * diag + model.aabb_min)
        for level in range(3):
            s = 2.0 ** level
            planes = [[((k / 128.0 - 0.5) * s + 0.5) for k in range(int(np.floor(((lo_w[a] - 0.5) / s + 0.5) * 128)), int(np.ceil(((hi_w[a] - 0.5) / s + 0.5) * 128)) + 1)]
                      for a in range(3)]
            planes = [[_to_warped(model, np.full(3, x, F32))[a] for x in pl[:: max(1, len(pl) // 6)]] for a, pl in enumerate(planes)]
            pts.append(_on_planes(rng, lo, hi, planes, 12))
        # cascade boundaries (world |p - 0.5| = 0.5, 1, 2) and the train AABB's faces
        pts.append(_on_planes(rng, lo, hi, _world_planes(model, lo_w, hi_w, [-1.5, -0.5, 0.0, 1.0, 1.5, 2.5]), 60))
        # random points inside and around the operator
        mid, ext = (lo + hi) / 2, (hi - lo) / 2
        pts.append((mid + (rng.random((n_random, 3)) * 2 - 1) * ext * 1.3).astype(F32))
    w = _ulp_neighbours(np.concatenate(pts))
    n = w.shape[0]
    c = np.zeros((n, 7), F32)
    c[:, :3] = w
    c[:, 3] = rng.random(n, dtype=F32)
    d = rng.standard_normal((n, 3))
    c[:, 4:] = ((d / np.linalg.norm(d, axis=1, keepdims=True) + 1) * 0.5).astype(F32)
    return c


# ---- the LUT-free rule ---------------------------------------------------------------------------------------------------------
def _cage_lut_free(op, pw, dw, empty, tet, n_in, chunk=2048):
    """interpolate_tet on rows pw [n, 3], dw [n, 3] (updated in place), empty [n] (only set); tet [n] receives the tet that mapped each
    row and n_in [n] how many tets contained it (rows this cage maps only)."""
    host, _ = op.to_op()
    mn, mx = op.aabb_min.astype(F32), op.aabb_max.astype(F32)
    diag = (mx - mn).astype(F32)
    wb = (_v(host.warped_bbox_min), _v(host.warped_bbox_max))
    ob = (_v(host.original_warped_bbox_min), _v(host.original_warped_bbox_max))
    V = op.vertices[op.tets].astype(F32)  # [T, 4, 3]
    O = op.original_vertices[op.tets].astype(F32)
    in_def = np.zeros(pw.shape[0], bool)
    rows = np.nonzero(((pw >= wb[0]) & (pw <= wb[1])).all(1))[0]
    with np.errstate(all="ignore"):
        for s in range(0, rows.size, chunk):
            r = rows[s: s + chunk]
            p = fma(pw[r], diag, mn)[:, None, :]   # [m, 1, 3]
            a, b, c, d = V[None, :, 0], V[None, :, 1], V[None, :, 2], V[None, :, 3]
            inside = same_side(a, b, c, d, p) & same_side(b, c, d, a, p) & same_side(c, d, a, b, p) & same_side(d, a, b, c, p)
            hit = inside.any(1)
            t = inside.argmax(1)                     # the lowest-index containing tet
            n_in[r[hit]] = inside.sum(1)[hit]
            tet[r[hit]] = t[hit]
            r, t, p = r[hit], t[hit], p[hit, 0]
            a, b, c, d = V[t, 0], V[t, 1], V[t, 2], V[t, 3]
            vap, vbp, vab, vac, vad, vbc, vbd = p - a, p - b, b - a, c - a, d - a, c - b, d - b
            v6 = (1.0 / stp(vab, vac, vad).astype(F64)).astype(F32)
            bary = [stp(vbp, vbd, vbc) * v6, stp(vap, vac, vad) * v6, stp(vap, vad, vab) * v6, stp(vap, vab, vac) * v6]
            bary = [x.astype(F32)[:, None] for x in bary]
            Ot = O[t]
            canon = fma(bary[3], Ot[:, 3], fma(bary[2], Ot[:, 2], fma(bary[0], Ot[:, 0], (bary[1] * Ot[:, 1]).astype(F32))))
            pw[r] = ((canon - mn) / diag).astype(F32)
            if op.use_local_rotations:
                R = op.rotations[t]                   # column-major 3x3 per row
                ud = fma(dw[r], F32(2.0), F32(-1.0))
                rd = np.stack([fma(R[:, k], ud[:, 0], fma(R[:, 3 + k], ud[:, 1], (R[:, 6 + k] * ud[:, 2]).astype(F32))) for k in range(3)], -1)
                dw[r] = ((rd + F32(1.0)) * F32(0.5)).astype(F32)
            in_def[r] = True
    if not op.copy:
        m = ~in_def & ((pw >= ob[0]) & (pw <= ob[1])).all(1)
        if m.any():
            p = fma(pw[m], diag, mn)
            level = mip_from_pos(p)
            bits = np.unpackbits(op.original_bitfield, bitorder="little")
            hit = bits[level.astype(np.int64) * 128 ** 3 + cell_index(p, level).astype(np.int64)].astype(bool)
            idx = np.nonzero(m)[0][hit]
            empty[idx] = True


def _abox_contains(b, p):
    mn, u, v, w = _v(b.min), _v(b.u), _v(b.v), _v(b.w)
    q = p - mn
    du, dv, dw = dot3(u[None], q), dot3(v[None], q), dot3(w[None], q)
    return (du >= 0) & (du < dot3(u, u)) & (dv >= 0) & (dv < dot3(v, v)) & (dw >= 0) & (dw < dot3(w, w))


def _mat_t_vec(M, v):
    return np.stack([fma(M[3 * k], v[:, 0], fma(M[3 * k + 1], v[:, 1], (M[3 * k + 2] * v[:, 2]).astype(F32))) for k in range(3)], -1)


def _affine_lut_free(host, pw, dw, empty):
    """translate_in_box on rows pw, dw (updated in place), empty (only set)."""
    M = _v(host.rotation)
    inside = _abox_contains(host.destination_box, pw)
    c = _v(host.destination_box.center)
    q = ((pw[inside] - c) / _v(host.scale)).astype(F32)
    pw[inside] = ((_mat_t_vec(M, q) + c).astype(F32) - _v(host.translation)).astype(F32)
    if host.correct_dir:
        dw[inside] = ((_mat_t_vec(M, fma(dw[inside], F32(2.0), F32(-1.0))) + F32(1.0)) * F32(0.5)).astype(F32)
    if host.hide_original:
        empty |= ~inside & _abox_contains(host.selection_box, pw)


def map_rays_lut_free(items, coords, want_tets=False):
    """EditOperator::map_rays of every item, reverse list order, without the lookup table: (coords [n, 7], empty mask uint8 [n]).
    want_tets: also (tet, n_in), per row the tet of the last cage that mapped it (-1: none) and how many of that cage's tets contain it."""
    c = np.ascontiguousarray(coords, F32).copy()
    pw, dw = c[:, :3].copy(), c[:, 4:].copy()
    empty = np.zeros(c.shape[0], bool)
    tet, n_in = np.full(c.shape[0], -1, np.int64), np.zeros(c.shape[0], np.int64)
    for it in reversed(items):
        if isinstance(it, EmptyOp):
            continue
        if isinstance(it, editing.CageDeformation):
            _cage_lut_free(it, pw, dw, empty, tet, n_in)
        else:
            _affine_lut_free(it.to_op()[0], pw, dw, empty)
    c[:, :3], c[:, 4:] = pw, dw
    return (c, empty.astype(np.uint8)) + ((tet, n_in) if want_tets else ())

