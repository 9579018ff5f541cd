"""CPU checks of the density input gradient restatement and of the mesh optimisation step mirror (oracle/mesh_opt_oracle.cpp).

* The float64 analytic gradient (chain rule through the density MLP and the hash grid, with tcnn's 128 seed and 1/128) matches central
  finite differences of the float64 encode + density MLP, at points away from cell boundaries and ReLU kinks.
* The fp32 restatement the GPU is held to agrees with the float64 gradient up to its fp16 rounding.
* The step mirror's Adam skips coordinates whose gradient is 0 and keeps one step counter per coordinate.
"""
import ctypes as C

import numpy as np

from conftest import random_coords


def _levels(model):
    from oracle import oracle as orc

    n = model.desc.n_levels
    scale, res, off, size = np.zeros(n, np.float32), np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    assert orc.lib().orc_level_table(C.byref(model.desc), *[a.ctypes.data_as(C.c_void_p) for a in (scale, res, off, size)]) == 0
    return scale


def test_analytic_gradient_matches_central_differences(scene, oracle):
    from oracle import mesh_opt_oracle as mo

    model, _ = scene
    rng = np.random.default_rng(5)
    pos = 0.2 + 0.6 * rng.random((400, 3))
    # away from cell boundaries at every level: the fractional cell position is at least 1e-3 from 0 and 1
    frac = (pos[:, None, :] * _levels(model)[None, :, None].astype(np.float64) + 0.5) % 1.0
    pos = pos[(np.minimum(frac, 1 - frac) > 1e-3).all((1, 2))]
    assert pos.shape[0] > 20
    h = 1e-7
    dens, grad = mo.density_f64(oracle, pos)
    fd = np.zeros_like(grad)
    one_sided = np.zeros_like(grad)
    for d in range(3):
        e = np.zeros(3)
        e[d] = h
        fp, _ = mo.density_f64(oracle, pos + e, False)
        fm, _ = mo.density_f64(oracle, pos - e, False)
        fd[:, d] = (fp - fm) / (2 * h)
        one_sided[:, d] = np.abs((fp - dens) - (dens - fm)) / h
    scale = np.abs(grad).max(1)
    # away from ReLU kinks: the two one-sided slopes agree (a kink within h changes one of them by a finite amount)
    smooth = (one_sided < 1e-5 * np.maximum(scale, 1.0)[:, None]).all(1)
    assert smooth.sum() > 20
    assert (scale[smooth] > 1e-3).all()
    err = np.abs(grad - fd).max(1) / scale
    assert err[smooth].max() < 1e-6, err[smooth].max()


def test_fp32_restatement_follows_the_float64_gradient(scene, oracle):
    from oracle import mesh_opt_oracle as mo

    coords = random_coords(2000, seed=3)
    g32, _, _ = mo.density_gradient(oracle, coords)
    _, g64 = mo.density_f64(oracle, coords[:, :3].astype(np.float64))
    scale = np.abs(g64).max(1)
    err = np.abs(g32 - g64).max(1) / np.maximum(scale, 1e-3)
    # fp16 features, activations and dfeat: per-mille differences, and a few points where fp16 rounding flips a ReLU
    assert np.median(err) < 5e-3 and (err < 5e-2).mean() > 0.98, (np.median(err), (err < 5e-2).mean())
    # the sign and the 1/128 scale: the two agree in direction on almost every point
    cos = (g32 * g64).sum(1) / (np.linalg.norm(g32, axis=1) * np.linalg.norm(g64, axis=1) + 1e-30)
    assert (cos > 0.99).mean() > 0.98


def _one_triangle():
    pos = np.zeros((128, 3), np.float32)
    pos[:3] = [[0.5, 0.5, 0.5], [0.6, 0.5, 0.5], [0.5, 0.6, 0.5]]
    return pos, np.array([[0, 1, 2]], np.uint32)


def test_adam_skips_zero_gradients_and_counts_steps_per_coordinate():
    from oracle import mesh_opt_oracle as mo

    pos, F = _one_triangle()
    dens = np.full(128, np.float16(1.0)).view(np.uint16)  # above thresh 0: sign +1
    # density term only: the opt gradient of a vertex is normalize(grad), so a zero component of grad is an exactly zero gradient
    g1 = np.tile(np.float32([1.0, 0.0, 0.0]), (128, 1))
    p1, n1, st = mo.mesh_opt_step(pos, F, dens, g1, 0.0, 0.0, 1.0, 0.0)
    m1, m2, steps = st
    assert (steps[:, 0] == 1).all() and (steps[:, 1:] == 0).all()
    assert (m1[:, 1:] == 0).all() and (m2[:, 1:] == 0).all()
    assert (p1[:, 1:] == pos[:, 1:]).all()
    # Adam's first step moves by lr = 1e-4 against the gradient's sign
    np.testing.assert_allclose(pos[:, 0] - p1[:, 0], 1e-4, rtol=1e-3)
    g2 = np.tile(np.float32([0.0, 1.0, 0.0]), (128, 1))
    p2, n2, st = mo.mesh_opt_step(p1, F, dens, g2, 0.0, 0.0, 1.0, 0.0, st)
    m1, m2, steps = st
    assert (steps[:, 0] == 1).all() and (steps[:, 1] == 1).all() and (steps[:, 2] == 0).all()
    assert (p2[:, 0] == p1[:, 0]).all() and (p2[:, 2] == pos[:, 2]).all()
    # y's first step is a first step again (its own counter): the debiased step is lr, not the 0.74 lr of a shared counter at t = 2
    np.testing.assert_allclose(p1[:, 1] - p2[:, 1], 1e-4, rtol=1e-3)
    # the normals are the 1-ring of the positions the step read: (pb - pa) x (pa - pc) of the one triangle on its three vertices
    pa, pb, pc = pos[0].astype(np.float64), pos[1].astype(np.float64), pos[2].astype(np.float64)
    np.testing.assert_allclose(n1[:3], np.tile(np.cross(pb - pa, pa - pc), (3, 1)), rtol=1e-6)
    assert (n1[3:] == 0).all()


def test_step_mirror_smoothing_moves_towards_the_centroid():
    from oracle import mesh_opt_oracle as mo

    pos, F = _one_triangle()
    dens = np.zeros(128, np.uint16)
    grad = np.zeros((128, 3), np.float32)
    p1, _, _ = mo.mesh_opt_step(pos, F, dens, grad, 0.0, 1.0, 0.0, 0.0)
    # vertex 1's centroid is (pos0 + pos2) / 2 = (0.5, 0.55, 0.5): x decreases, y increases, z has a zero gradient and stays
    assert p1[1, 0] < pos[1, 0] and p1[1, 1] > pos[1, 1] and p1[1, 2] == pos[1, 2]
    # padding rows: no triangles, centroid at the origin, at the origin already: zero gradient, they stay
    assert (p1[3:] == 0).all()
