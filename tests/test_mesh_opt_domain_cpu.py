"""The mesh-optimisation oracle (oracle/mesh_opt_oracle.cpp) over its whole domain, without a GPU.

* On every grid geometry of tests/encoding_domain.py, inside and outside the unit cube (dense levels wrap there; the field is still
  piecewise smooth): the float64 analytic gradient matches central differences away from cell boundaries and ReLU kinks, and the fp32
  restatement the device is held to follows the float64 gradient under both accumulator policies.
* The step mirror's Adam over hundreds of steps, with zero gradients interleaved per coordinate, equals a numpy transcription of tcnn's
  adam_step (fp32 roundings as written, fmaf correctly rounded) fed the same table of debiasing powers; without a table it is the host's powf.
* The sign rule of the density term on NaN differences is the device's: +1 for +NaN and -NaN thresholds alike.
"""
import ctypes as C

import numpy as np
import pytest

import encoding_domain as ed
import mesh_opt_domain as mod
from edit_domain import fma

F32 = np.float32


def _scale(d):
    from oracle import oracle as orc

    n = d.n_levels
    scale, res, off, size = np.zeros(n, np.float32), np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    assert orc.lib().orc_level_table(C.byref(d), *[a.ctypes.data_as(C.c_void_p) for a in (scale, res, off, size)]) == 0
    return scale


def _oracle(name):
    from oracle import oracle as orc

    d = ed.GEOMETRIES[name]
    return d, orc.Oracle(d, ed.make_model(d, seed=5), None)


@pytest.mark.parametrize("name", list(ed.GEOMETRIES))
def test_analytic_gradient_matches_central_differences_on_every_geometry(name):
    from oracle import mesh_opt_oracle as mo

    d, o = _oracle(name)
    rng = np.random.default_rng(11)
    # inside the cube, past it on every side, and far out (where the dense levels wrap and the float->int conversion saturates)
    pos = np.concatenate([rng.random((300, 3)), rng.uniform(-2.5, 3.5, (300, 3)), rng.uniform(-1e3, 1e3, (60, 3))])
    scale = _scale(d).astype(np.float64)
    frac = (pos[:, None, :] * scale[None, :, None] + 0.5) % 1.0
    pos = pos[(np.minimum(frac, 1 - frac) > 1e-3).all((1, 2))]
    assert pos.shape[0] > 50 and (np.abs(pos - 0.5) > 0.5).any(1).sum() > 20
    h = 1e-7
    dens, grad = mo.density_f64(o, pos)
    fd, one_sided = np.zeros_like(grad), np.zeros_like(grad)
    for k in range(3):
        e = np.zeros(3)
        e[k] = h
        fp, _ = mo.density_f64(o, pos + e, False)
        fm, _ = mo.density_f64(o, pos - e, False)
        fd[:, k] = (fp - fm) / (2 * h)
        one_sided[:, k] = np.abs((fp - dens) - (dens - fm)) / h
    mag = np.abs(grad).max(1)
    smooth = (one_sided < 1e-5 * np.maximum(mag, 1.0)[:, None]).all(1)
    assert smooth.sum() > 40, smooth.sum()
    assert (mag[smooth] > 1e-3).mean() > 0.9
    err = np.abs(grad - fd).max(1) / np.maximum(mag, 1e-2)
    # far out, the cell position scale * x + 0.5 keeps fewer fractional bits in float64 and the differences are noisier by that much
    far = np.abs(pos).max(1) > 10
    assert (smooth & far).sum() > 10
    print(f"\n{name}: {smooth.sum()} smooth points, max relative error {err[smooth & ~far].max():.2e}, {err[smooth & far].max():.2e} far out")
    assert err[smooth & ~far].max() < 1e-7 and err[smooth & far].max() < 1e-5


@pytest.mark.parametrize("policy", [0, 1], ids=["f32", "f16"])
@pytest.mark.parametrize("name", list(ed.GEOMETRIES))
def test_fp32_restatement_follows_the_float64_gradient_on_every_geometry(name, policy):
    from conftest import random_coords
    from oracle import mesh_opt_oracle as mo

    d, o = _oracle(name)
    coords = random_coords(3000, seed=3)
    coords[1500:, :3] = np.random.default_rng(4).uniform(-0.5, 1.5, (1500, 3)).astype(F32)  # past the cube
    old = mo.set_mlp_policy(policy)
    try:
        g32, _, _ = mo.density_gradient(o, coords)
    finally:
        mo.set_mlp_policy(old)
    _, g64 = mo.density_f64(o, coords[:, :3].astype(np.float64))
    mag = np.abs(g64).max(1)
    live = mag > 1e-2  # a gradient that fp16 rounding can zero out carries no direction to compare
    assert live.mean() > 0.5
    err = np.abs(g32 - g64).max(1)[live] / mag[live]
    cos = ((g32 * g64).sum(1) / (np.linalg.norm(g32, axis=1) * np.linalg.norm(g64, axis=1) + 1e-30))[live]
    print(f"\n{name}: median relative error {np.median(err):.2e}, {100 * (err < 5e-2).mean():.2f} % under 5e-2, {100 * (cos > 0.99).mean():.2f} % cos > 0.99")
    # fp16 features, activations and dfeat: per-mille differences, and a few points where fp16 rounding flips a ReLU. Levels of 2^16 cells
    # and more per unit (aabb128) also round the cell position fma(scale, x, 0.5) to 1/128 of a cell or coarser in fp32, which moves their
    # interpolation weights by that much: measured 92 % under 5e-2 and 95 % of the directions within cos 0.99 there.
    coarse = float(_scale(d).max()) >= 2.0 ** 16
    assert np.median(err) < 5e-3 and (err < 5e-2).mean() > (0.9 if coarse else 0.97)
    assert (cos > 0.99).mean() > (0.93 if coarse else 0.97)


# ---- Adam over many steps --------------------------------------------------------------------------------------------------------
def _adam_transcription(x, grads, pows):
    """tcnn's adam_step on non-matrix parameters, step by step in numpy: fp32 roundings where the CUDA source rounds, fmaf where nvcc
    contracts (the moment updates and the final subtraction), each coordinate skipped while its gradient is 0 and counted on its own."""
    x = x.astype(F32).copy()
    m1, m2 = np.zeros_like(x), np.zeros_like(x)
    t = np.zeros(x.shape, np.int64)
    b1, b2, lr0, eps = F32(0.9), F32(0.99), F32(1e-4), F32(1e-8)
    for g in grads:
        live = g != 0  # coordinates that never stepped read row 0 of the table and divide 0 by 0; np.where drops them
        nm1 = fma(b1, m1, (F32(1) - b1) * g)
        nm2 = fma(b2, m2, (F32(1) - b2) * (g * g))
        m1, m2 = np.where(live, nm1, m1), np.where(live, nm2, m2)
        t = t + live
        p1, p2 = pows[t, 0], pows[t, 1]
        with np.errstate(invalid="ignore", divide="ignore"):
            lr = lr0 * (np.sqrt(F32(1) - p2) / (F32(1) - p1))
            eff = lr / (np.sqrt(m2) + eps)
        x = np.where(live, fma(-eff, m1, x), x)
    return x, m1, m2, t


def _gradient_sequence(steps, rows, seed=3):
    rng = np.random.default_rng(seed)
    g = (rng.standard_normal((steps, rows, 3)) * np.exp(rng.uniform(-8, 4, (steps, rows, 3)))).astype(F32)
    g[rng.random(g.shape) < 0.25] = 0.0  # zeros interleaved per coordinate
    g[:, 0, 1] = 0.0                       # one coordinate never moves
    g[: steps // 2, 1] = 0.0                # one row starts late: its first step is t = 1 again
    return g


@pytest.mark.parametrize("table", ["float64", "host_powf"])
def test_mirror_adam_over_many_steps_equals_the_transcription(table):
    from oracle import mesh_opt_oracle as mo

    steps, rows = 440, 128
    n = steps + 2
    if table == "host_powf":
        pows = mod.host_pows(n)
    else:  # float64 powers rounded once, which differ from glibc's powf at some t: the mirror must read the table, not call powf
        tt = np.arange(n, dtype=np.float64)
        pows = np.stack([np.float64(F32(0.9)) ** tt, np.float64(F32(0.99)) ** tt], 1).astype(F32)
        assert (pows != mod.host_pows(n)).any()
    x0 = np.random.default_rng(1).uniform(-2, 2, (rows, 3)).astype(F32)
    grads = _gradient_sequence(steps, rows)
    want, wm1, wm2, wt = _adam_transcription(x0, grads, pows)
    x, st = x0, None
    for g in grads:
        x, st = mo.adam_step(x, g, st, pows=pows)
    np.testing.assert_array_equal(st[2], wt)
    assert wt.max() >= 300 and wt[0, 1] == 0 and (wt[1] <= steps - steps // 2).all()
    np.testing.assert_array_equal(st[0].view(np.uint32), wm1.view(np.uint32))
    np.testing.assert_array_equal(st[1].view(np.uint32), wm2.view(np.uint32))
    np.testing.assert_array_equal(x.view(np.uint32), want.view(np.uint32))
    if table == "host_powf":  # no table: the host's powf, the same bytes
        x2, st2 = x0, None
        for g in grads:
            x2, st2 = mo.adam_step(x2, g, st2)
        np.testing.assert_array_equal(x2.view(np.uint32), x.view(np.uint32))


def test_mirror_step_through_many_steps_reads_the_table():
    """orc_mesh_opt_step takes the same table: the density term alone with a constant unit gradient moves each coordinate by exactly
    Adam's debiased step, which depends on the powers at every t."""
    from oracle import mesh_opt_oracle as mo

    pos = np.zeros((128, 3), F32)
    pos[:3] = [[0.5, 0.5, 0.5], [0.6, 0.5, 0.5], [0.5, 0.6, 0.5]]
    F = np.array([[0, 1, 2]], np.uint32)
    dens = np.full(128, np.float16(1.0)).view(np.uint16)
    grad = np.tile(F32([1.0, -1.0, 0.0]), (128, 1))
    n = 320
    a, b = mod.host_pows(n + 1), mod.host_pows(n + 1)
    b[1:, 1] *= F32(1 - 1e-3)  # a different table: the positions must move differently
    out = []
    for pows in (a, b):
        p, st = pos, None
        for _ in range(n):
            p, _, st = mo.mesh_opt_step(p, F, dens, grad, 0.0, 0.0, 1.0, 0.0, st, pows=pows)
        assert (st[2][:, :2] == n).all() and (st[2][:, 2] == 0).all()
        out.append(p)
    assert (out[0][:, :2] != out[1][:, :2]).any() and (out[0][:, 2] == pos[:, 2]).all()
    with pytest.raises(AssertionError):  # a table shorter than the step count is an error, not a silent fallback
        mo.mesh_opt_step(pos, F, dens, grad, 0.0, 0.0, 1.0, 0.0, None, pows=a[:1])


def test_density_sign_of_a_nan_difference_is_positive():
    """dens - thresh is NaN for a NaN threshold: the device's canonical NaN has its sign bit clear, so the density term pushes as for a
    positive difference whether the threshold is +NaN or -NaN."""
    from oracle import mesh_opt_oracle as mo

    pos = np.zeros((128, 3), F32)
    pos[:3] = [[0.5, 0.5, 0.5], [0.6, 0.5, 0.5], [0.5, 0.6, 0.5]]
    F = np.array([[0, 1, 2]], np.uint32)
    dens = np.full(128, np.float16(-1.0)).view(np.uint16)
    grad = np.tile(F32([1.0, 2.0, -3.0]), (128, 1))
    assert np.signbit(F32(mod.NEG_NAN)) and np.isnan(mod.NEG_NAN)
    _, _, g_pos = mo.mesh_opt_gradient(pos, F, dens, grad, 10.0, 0.0, 1.0, 0.0)  # -1 - 10 < 0: sign -1
    for t in (np.nan, mod.NEG_NAN):
        _, _, g = mo.mesh_opt_gradient(pos, F, dens, grad, t, 0.0, 1.0, 0.0)
        np.testing.assert_array_equal(g.view(np.uint32), (-g_pos).view(np.uint32))
