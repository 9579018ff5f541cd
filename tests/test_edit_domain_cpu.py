"""CPU: the edit operators over their whole domain (tests/edit_domain.py), for every operator set.

- The oracle's map_rays equals the LUT-free rule bit for bit, except where the lookup table does not list a tet that the fp32 point-in-tet
  test accepts; the reference build (or its stored results) shows the same miss on those samples, so it is recorded as reference behaviour.
- A float64 check that does not depend on fp32 emulation: a sample at least DELTA from every tet face lies in exactly one tet (outside
  folds), and the oracle maps it to that tet's float64 barycentric image within BOUND.
- The oracle's map_positions / compute_poisson_residual_density / compute_poisson_full_residuals against the reference's own
  EditOperator overrides (oracle/ref_driver.cpp), stored under tests/golden/ref/ where the reference is absent.
"""
import numpy as np
import pytest

import edit_domain as ed
from oracle import oracle as orc
from ref_golden import ref

F32, F64 = np.float32, np.float64
DELTA = 1e-4  # world units: far enough from every face that fp32 sign tests cannot disagree with float64
BOUND = 2e-6  # warped units (1.7e-5 world on the 4-unit train AABB): a few fp32 ulps of the canonical position, times the tets' conditioning


def _oracle(scene, ops):
    model, occ = scene
    return orc.Oracle(model.desc, model.params, occ, ops)


@pytest.mark.parametrize("name", ed.NAMES)
def test_oracle_map_rays_equals_the_lut_free_rule(scene, name):
    model, occ = scene
    items = ed.build(model, name)
    c = ed.samples(model, items)
    co, mo = _oracle(scene, ed.ops_of(items)).map_rays(c)
    cl, ml, tet, n_in = ed.map_rays_lut_free(items, c, want_tets=True)
    moved = (cl[:, :3] != c[:, :3]).any(1)
    assert moved.sum() > 1000, moved.sum()
    if ed.cages_of(items):
        # premise: samples on shared faces (two or more tets contain them) are mapped
        assert (n_in >= 2).sum() > 40, (n_in >= 2).sum()
    both_nan = np.isnan(co) & np.isnan(cl)
    differ = ((co.view(np.uint32) != cl.view(np.uint32)) & ~both_nan).any(1) | (mo != ml)
    if name == "flattened":
        assert np.isnan(co[:, :3]).any(1).sum() > 100  # the flat tet's barycentrics are 0 * inf
    rows = np.nonzero(differ)[0]
    if rows.size:
        # only lookup-table misses: the oracle found no tet in the sample's cell list, the LUT-free rule found one that the list lacks
        assert rows.size <= max(2, c.shape[0] // 5000), rows.size
        cage = ed.cages_of(items)[-1]
        assert len(ed.cages_of(items)) == 1, "a miss in a multi-cage set would need the cage it happened in"
        assert not (co[rows, :3] != c[rows, :3]).any(), "the oracle mapped a sample differently, not a lookup-table miss"
        p = ed.fma(c[rows, :3], model.aabb_max - model.aabb_min, model.aabb_min)
        level = ed.mip_from_pos(p)
        cell = level.astype(np.int64) * 128 ** 3 + ed.cell_index(p, level)
        for r, k, t in zip(rows, cell, tet[rows]):
            listed = cage.lut_idx[cage.lut_offsets[k]: cage.lut_offsets[k + 1]]
            assert t >= 0 and t not in listed, (r, t, listed)
        cr, mr = ref.map_rays(ed.ops_of(items), c[rows])
        assert np.array_equal(cr.view(np.uint32), co[rows].view(np.uint32)) and np.array_equal(mr, mo[rows]), "the reference maps these samples"


def _faces_distance(V, p):
    """float64: signed distances [n, T, 4] of p [n, 3] to the four faces of tets V [T, 4, 3], positive inside; and [T] volumes."""
    faces = ((1, 2, 3, 0), (0, 2, 3, 1), (0, 1, 3, 2), (0, 1, 2, 3))
    out = []
    for a, b, c, d in faces:
        n = np.cross(V[:, b] - V[:, a], V[:, c] - V[:, a])
        n /= np.linalg.norm(n, axis=1, keepdims=True)
        s = np.sign(np.einsum("tk,tk->t", n, V[:, d] - V[:, a]))
        out.append(np.einsum("tk,ntk->nt", n * s[:, None], p[:, None, :] - V[None, :, a]))
    vol = np.einsum("tk,tk->t", V[:, 1] - V[:, 0], np.cross(V[:, 2] - V[:, 0], V[:, 3] - V[:, 0])) / 6
    return np.stack(out, -1), vol


@pytest.mark.parametrize("name", [n for n in ed.NAMES if n != "flattened"])  # a flat tet has no face normal; the LUT-free test covers it
def test_float64_barycentric_image(scene, name):
    """Each cage alone: samples DELTA inside exactly one tet (and DELTA from every other tet's faces) map to its float64 barycentric image."""
    model, occ = scene
    items = ed.build(model, name)
    cages = ed.cages_of(items)
    if not cages:
        pytest.skip("no cage in this set")
    c = ed.samples(model, items)
    diag = (model.aabb_max - model.aabb_min).astype(F64)
    for cage in cages:
        co, _ = _oracle(scene, [cage.to_op()]).map_rays(c)
        p = ed.fma(c[:, :3], model.aabb_max - model.aabb_min, model.aabb_min).astype(F64)
        V = cage.vertices[cage.tets].astype(F64)
        keep = np.ones(c.shape[0], bool)
        checked = 0
        for s in range(0, c.shape[0], 2048):
            dist, vol = _faces_distance(V, p[s: s + 2048])
            inside = (dist > DELTA).all(-1)
            clear = (np.abs(dist) > DELTA).all(-1).all(-1)
            one = clear & (inside.sum(1) == 1)
            keep[s: s + 2048] = one
            r = np.nonzero(one)[0]
            if r.size == 0:
                continue
            t = inside[r].argmax(1)
            # barycentric coordinates in float64 by solving the 3x3 system, then the canonical position
            A = np.stack([V[t, 1] - V[t, 0], V[t, 2] - V[t, 0], V[t, 3] - V[t, 0]], -1)
            lam = np.linalg.solve(A, (p[s + r] - V[t, 0])[..., None])[..., 0]
            O = cage.original_vertices[cage.tets[t]].astype(F64)
            canon = O[:, 0] + np.einsum("nk,nkj->nj", lam, O[:, 1:] - O[:, :1])
            want = (canon - model.aabb_min) / diag
            err = np.abs(co[s + r, :3] - want).max(1)
            assert err.max() <= BOUND, (name, int(s + r[err.argmax()]), float(err.max()))
            checked += r.size
        # premise: enough samples checked, and a missing tet would show (an unmapped sample is far from its image)
        assert checked > 500, checked
        assert (np.abs(co[keep, :3] - c[keep, :3]).max(1) > 10 * BOUND).sum() > 0.5 * checked or name == "no_tets"


def _subsample(c, k, seed):
    rows = np.sort(np.random.default_rng(seed).choice(c.shape[0], min(k, c.shape[0]), replace=False))
    return np.ascontiguousarray(c[rows])


@pytest.mark.skipif(not ref.usable("test_edit_domain_cpu"), reason="no reference build and no stored reference results")
@pytest.mark.parametrize("name", ed.NAMES)
def test_map_positions_and_residual_density_vs_reference(scene, name):
    """CageDeformation / AffineDuplication ::map_positions and ::compute_poisson_residual_density of the reference, and its
    compute_poisson_full_residuals on the membrane sets. Positions: the reference's CPU build contracts dot and cross products
    differently from nvcc (which the oracle follows bit for bit), so a sample exactly on a tet or box face may be decided the other way:
    such samples jump (more than 8 ulp) and are bounded in number; every other position is within 8 ulp, the bar of the map_rays pin in
    test_oracle_vs_ref.py (ulps of the warped value). The residual density is added to the same positions on both sides and agrees bit for bit."""
    model, occ = scene
    items = ed.build(model, name)
    ops = ed.ops_of(items)
    o = _oracle(scene, ops)
    c = _subsample(ed.samples(model, items), 1500, 1)  # stride 7: the position is the first 3 of each NerfCoordinate row
    mask0 = np.zeros(c.shape[0], np.uint8)
    po, mo = o.map_positions(c, mask0)
    pr, mr = ref.map_positions(ops, c, mask0)
    assert (po[:, :3] != c[:, :3]).any(1).sum() > 150
    assert np.array_equal(po[:, 3:], c[:, 3:]) and np.array_equal(pr[:, 3:], c[:, 3:])  # only the position moves
    assert (mo != mr).sum() <= 2
    both_nan = np.isnan(po[:, :3]) & np.isnan(pr[:, :3])
    ulp = np.where(both_nan, 0, np.abs(po[:, :3].view(np.int32).astype(np.int64) - pr[:, :3].view(np.int32)))
    jumps = (ulp > 8).any(1)
    assert jumps.sum() <= max(5, c.shape[0] // 200), jumps.sum()
    assert ulp[~jumps].max() <= 8
    h = np.random.default_rng(2).uniform(-3.0, 20.0, c.shape[0]).astype(np.float16).view(np.uint16)
    ho = o.poisson_residual_density(po, h)
    hr = ref.poisson_residual_density(ops, po, h)
    assert np.array_equal(ho, hr)
    has_rd = [cg.apply_poisson and cg.boundary_residual_density is not None for cg in ed.cages_of(items)]
    assert ((ho != h).sum() > 300) == any(has_rd)
    if any(cg.boundary_shs is not None or cg.boundary_residual_density is not None for cg in ed.cages_of(items)):
        cp = _subsample(c, 400, 3)
        sh_o, od_o, rd_o = o.poisson_residuals(cp)
        sh_r, od_r, rd_r = ref.poisson_residuals(ops, cp)
        assert np.array_equal(od_o != 0, od_r != 0) and np.array_equal(rd_o != 0, rd_r != 0)
        assert np.allclose(od_o, od_r, rtol=2e-5, atol=1e-5) and np.allclose(rd_o, rd_r, rtol=2e-5, atol=1e-5) and np.allclose(sh_o, sh_r, rtol=2e-5, atol=2e-5)


@pytest.mark.parametrize("arrays", [("shs",), ("od",), ("rd",), ("shs", "od"), ("shs", "rd"), ("od", "rd")])
def test_partial_membrane_gating(scene, arrays):
    """A cage with only some membrane arrays: the full residuals (render) skip it unless all three are present (cage_deformation.cu:686);
    the density residual (occupancy update) uses it whenever boundary_residual_density is present (:650). The oracle's grid update and
    its residual-density entry point are one implementation."""
    model, occ = scene
    cage = ed.with_membrane(ed.dyadic_cage(model, (0.5, 0.625, 0.75), (0.125, 0.125, 0.125)), 12, arrays=arrays, amplitude=1.5)
    o = _oracle(scene, [cage.to_op()])
    c = ed.samples(model, [cage])
    sh, od, rd = o.poisson_residuals(c)
    assert not od.any() and not rd.any() and not sh.any()
    h = np.full(c.shape[0], 0x3C00, np.uint16)  # 1.0
    added = o.poisson_residual_density(c, h) != h
    assert added.sum() > 1000 if "rd" in arrays else not added.any()
