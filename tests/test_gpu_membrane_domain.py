"""The membrane boundary on the GPU over its whole domain (DESIGN §7 (f)-4).

nsb_poisson_boundary: k_boundary_fit against a float64 restatement of GrowingSelection::compute_poisson_boundary's device part
(activate_network_output, filter_empty and the SH9 fit of project_sh9, growing_selection.cu:2182-2218, 2323-2345, sh_utils.cu). The
restatement reads the oracle's boundary coordinates (the same pcg32 jitter as the product's host draw) and the device's own fp16 network
rows for them (nsb_inference), which are the rows k_boundary_fit consumes, so the MLP drops out and what is left is the kernel's own
arithmetic. With the identity and ReLU colour activations that arithmetic is also restated in float32, operation for operation, and must
match bit for bit: a coordinate of the oracle's draw that were not the product's would show there.

nsb_cage_set_membrane: k_membrane_blend over its launch shape (block (32, 4), (nv + 3) / 4 CTAs) and its degenerate inputs, bit for bit
against oracle.membrane_blend, and its non-NaN entries against a float64 model within a derived bound.
"""
import numpy as np
import pytest

import edit_fixtures as fx
from nerfshop_b200 import abi
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
U = 2.0 ** -24  # unit roundoff of float32
A = abi
TRAIN_AABB = ((-1.5, -1.5, -1.5), (2.5, 2.5, 2.5))


def _same(a, b):
    """Bit equality, a NaN on both sides counting as equal (the device's NaN payload is not the host's)."""
    a, b = np.asarray(a), np.asarray(b)
    both = np.isnan(a) & np.isnan(b)
    return np.array_equal(np.where(both, 0, a.view(np.uint32)), np.where(both, 0, b.view(np.uint32)))


@pytest.fixture
def policy(renderer, request):
    old = orc.set_mlp_policy(request.param)
    renderer.set_mlp_accumulator(request.param)
    yield request.param
    renderer.set_mlp_accumulator(1)
    orc.set_mlp_policy(old)


# ---- nsb_poisson_boundary ------------------------------------------------------------------------------------------------------------
def _points(model, kind, n):
    """World points: near the fox's surface (occupied cells), anywhere in the train AABB (mostly empty cells), outside it, and exactly
    on the cascade boundaries (a coordinate at 0.5 +- 0.5 * 2^k, k = 0..2, in every axis)."""
    rng = np.random.default_rng(n + 17 * len(kind))
    op = fx.e1(model)[0]
    occupied = np.concatenate([op.cage_original, op.vertices])
    parts = {
        "occupied": occupied[rng.integers(0, occupied.shape[0], n)],
        "aabb": rng.uniform(TRAIN_AABB[0], TRAIN_AABB[1], (n, 3)),
        "outside": np.where(rng.random((n, 3)) < 0.5, 1.0, -1.0) * rng.uniform(2.1, 5.0, (n, 3)) + 0.5,  # |p - 0.5| > 2: outside [-1.5, 2.5]
    }
    cascade = rng.uniform(-1.5, 2.5, (n, 3))
    edges = np.array([0.0, 1.0, -0.5, 1.5, -1.5, 2.5])
    ax = rng.integers(0, 3, n)
    cascade[np.arange(n), ax] = edges[rng.integers(0, edges.size, n)]
    parts["cascade"] = cascade
    if kind == "mixed":
        p = np.concatenate([parts[k] for k in ("occupied", "aabb", "outside", "cascade")])
        p = p[rng.permutation(p.shape[0])[:n]]
    else:
        p = parts[kind]
    return np.ascontiguousarray(p, F32)


# (sampling width, hemisphere width, rgb activation, density activation, is_inside, points, n): n * w^2 a multiple of 128 and not;
# every activation on each side at least once, with both paired once (logistic / exponential, the reference's defaults). A hemisphere
# width above the sampling width draws directions from part of the sphere; below it, acosf's argument leaves [-1, 1].
BOUNDARY_CASES = {
    "w1_inside_mixed23": (1, 1, A.NSB_ACT_LOGISTIC, A.NSB_ACT_EXPONENTIAL, True, "mixed", 23),
    "w2_hw5_none_none_1": (2, 5, A.NSB_ACT_NONE, A.NSB_ACT_NONE, False, "occupied", 1),
    "w7_relu_relu_inside_cascade23": (7, 7, A.NSB_ACT_RELU, A.NSB_ACT_RELU, True, "cascade", 23),
    "w10_logistic_exp_inside_mixed1000": (10, 10, A.NSB_ACT_LOGISTIC, A.NSB_ACT_EXPONENTIAL, True, "mixed", 1000),
    "w10_hw13_exp_logistic_aabb23": (10, 13, A.NSB_ACT_EXPONENTIAL, A.NSB_ACT_LOGISTIC, False, "aabb", 23),
    "w64_none_exp_inside_occupied23": (64, 64, A.NSB_ACT_NONE, A.NSB_ACT_EXPONENTIAL, True, "occupied", 23),
    "w64_hw91_relu_none_outside1": (64, 91, A.NSB_ACT_RELU, A.NSB_ACT_NONE, True, "outside", 1),
    "w7_hw9_exp_relu_inside_occupied1000": (7, 9, A.NSB_ACT_EXPONENTIAL, A.NSB_ACT_RELU, True, "occupied", 1000),
}

_SH_C = [F32(0.282095), F32(0.488603), F32(1.092548), F32(0.315392), F32(0.546274)]  # project_sh9's constants, float as it stores them


def _act64(v, act, rgb):
    """network_to_rgb / network_to_density (common_nerf.cu:38-66) in float64; v: the fp16 network output as float64. A colour's
    exponential clamps its argument to [-10, 10]."""
    if act == A.NSB_ACT_NONE:
        return v
    if act == A.NSB_ACT_RELU:
        return np.maximum(v, 0.0)
    if act == A.NSB_ACT_LOGISTIC:
        return 1.0 / (1.0 + np.exp(-v))
    return np.exp(np.clip(v, -10.0, 10.0) if rgb else v)


def _act_rel_err(v, act, rgb):
    """Relative error bound of the device's activation at v (CUDA C Programming Guide, maximum ulp errors of the single-precision
    functions): logistic 1/(1 + expf(-v)), expf within 2 ulp, then one rounding each for the sum and the division: 3 * 2^-23;
    exponential: __expf, within 2 + floor(|1.173 * v|) ulp, v clamped to [-10, 10] for colours (network_to_rgb)."""
    if act in (A.NSB_ACT_NONE, A.NSB_ACT_RELU):
        return np.zeros_like(v)
    if act == A.NSB_ACT_LOGISTIC:
        return np.full_like(v, 3 * 2.0 ** -23)
    x = np.clip(v, -10.0, 10.0) if rgb else v
    return (2.0 + np.floor(np.abs(1.173 * x))) * 2.0 ** -23


def _basis(d):
    """project_sh9's nine basis values (float64) and, per value, the magnitude its float32 evaluation rounds against
    (|c| * (3 z^2 + 1) for Y_20, |c| * (x^2 + y^2) for Y_22, |Y| otherwise). d: [..., 3] float64 of float32 directions."""
    x, y, z = d[..., 0], d[..., 1], d[..., 2]
    c = [F64(k) for k in _SH_C]
    b = np.stack([np.full_like(x, c[0]), c[1] * y, c[1] * z, c[1] * x, c[2] * x * y, c[2] * y * z, c[3] * (3 * z * z - 1), c[2] * x * z,
                  c[4] * (x * x - y * y)], -1)
    mag = np.abs(b)
    mag[..., 6] = c[3] * (3 * z * z + 1)
    mag[..., 8] = c[4] * (x * x + y * y)
    return b, mag


def _basis32(d):
    """k_boundary_fit's float32 basis, operation for operation (products left to right as the reference writes them)."""
    x, y, z = d[..., 0], d[..., 1], d[..., 2]
    c = _SH_C
    return np.stack([np.full_like(x, c[0]), c[1] * y, c[1] * z, c[1] * x, (c[2] * x) * y, (c[2] * y) * z, c[3] * ((F32(3) * z) * z - F32(1)),
                     (c[2] * x) * z, c[4] * (x * x - y * y)], -1)


@pytest.mark.parametrize("policy", [0, 1], indirect=True, ids=["wide", "half"])
@pytest.mark.parametrize("case", list(BOUNDARY_CASES))
def test_poisson_boundary_vs_float64(scene, renderer, oracle, policy, case):
    """k_boundary_fit against float64 on the device's own network rows: the same filtered (zero) densities; densities within the
    activation's documented ulp bound; SH within |err| <= scale * (gamma_n * sum|t| + sum|r| * (3u * mag + (u + act_err) * |Y|)) + 2u |SH|,
    n = n_sh samples summed in float32 (gamma_n = n u / (1 - n u)), t the terms r * Y, mag the magnitude each basis value is rounded
    against, act_err the activation's relative error, 2u the float32 scale and its product."""
    model, _ = scene
    w, hw, rgb_act, dens_act, inside, kind, n = BOUNDARY_CASES[case]
    pts = _points(model, kind, n)
    dens, shs, p = renderer.poisson_boundary(pts, is_inside=inside, seed=7 + n, sampling_width=w, hemisphere_width=hw, train_aabb=TRAIN_AABB,
                                             rgb_activation=rgb_act, density_activation=dens_act)
    _, _, coords = oracle.poisson_boundary(pts, p, want_coords=True)
    n_sh = w * w
    rows = renderer.inference(coords).view(np.float16).astype(F64)  # [16, n * n_sh]
    raw_rgb = rows[:3].reshape(3, n, n_sh).transpose(1, 2, 0)        # [n, n_sh, 3]
    raw_d = rows[3].reshape(n, n_sh)[:, 0]

    # filter_empty: which points the oracle's is_inside test drops (its density for an exponential activation is then exactly 0)
    q = abi.NsbBoundarySampling.from_buffer_copy(p)
    q.density_activation, q.sampling_width, q.hemisphere_width = A.NSB_ACT_EXPONENTIAL, 1, 1
    dropped = oracle.poisson_boundary(pts, q)[0] == 0 if inside else np.zeros(n, bool)
    d64 = np.where(dropped, 0.0, _act64(raw_d, dens_act, rgb=False))
    assert np.array_equal(dens == 0, d64.astype(F32) == 0), (case, np.flatnonzero((dens == 0) != (d64.astype(F32) == 0))[:8])
    if inside and kind == "mixed":
        assert dropped.any() and (~dropped).any(), "is_inside must keep some points and drop others"
    live = ~dropped
    bound = _act_rel_err(raw_d, dens_act, rgb=False) * np.abs(d64) + (2.0 ** -126 if dens_act == A.NSB_ACT_EXPONENTIAL else 0.0)  # __expf flushes
    derr = np.abs(dens.astype(F64) - d64)
    assert (derr[live] <= bound[live]).all(), (case, float((derr / np.maximum(bound, 1e-300))[live].max()))

    # SH9 in float64
    cw = coords.reshape(n, n_sh, 7)[..., 4:].astype(F64)
    d32 = (cw * 2.0 - 1.0).astype(F32)                              # unwarp_direction: fma(c, 2, -1), rounded once
    Y, mag = _basis(d32.astype(F64))                                # [n, n_sh, 9]
    r = _act64(raw_rgb, rgb_act, rgb=True)                                  # [n, n_sh, 3]
    t = r[..., :, None] * Y[..., None, :]                           # [n, n_sh, 3, 9]
    scale = 4.0 * np.pi / n_sh
    exact = scale * t.sum(1).reshape(n, 27)
    gamma_n = n_sh * U / (1 - n_sh * U)
    act_err = _act_rel_err(raw_rgb, rgb_act, rgb=True)
    per_term = np.abs(r)[..., :, None] * (3 * U * mag[..., None, :] + (U + act_err[..., :, None]) * np.abs(Y)[..., None, :])
    sh_bound = scale * (gamma_n * np.abs(t).sum(1) + per_term.sum(1)).reshape(n, 27) + 2 * U * np.abs(exact) + 1e-45
    err = np.abs(shs.astype(F64) - exact)
    worst = float((err / sh_bound).max())
    print(f"\n{case} ({'wide' if policy == 0 else 'half'} accumulators): n_sh {n_sh}, {n} points; SH max |err| {err.max():.3e}, "
          f"largest err/bound {worst:.3f} (bound at that entry {sh_bound.flat[np.argmax(err / sh_bound)]:.3e}); "
          f"density max err/bound {float((derr / np.maximum(bound, 1e-300))[live].max()) if live.any() else 0.0:.3f}")
    assert worst <= 1.0, case

    # the identity / ReLU colours: k_boundary_fit's float32 arithmetic, bit for bit
    if rgb_act in (A.NSB_ACT_NONE, A.NSB_ACT_RELU):
        r32 = r.astype(F32)
        b32 = _basis32(d32)
        acc = np.zeros((n, 3, 9), F32)
        for i in range(n_sh):
            acc = acc + (r32[:, i, :, None] * b32[:, i, None, :]) * F32(1.0)
        want = (acc.reshape(n, 27) * F32(scale)).astype(F32)
        assert _same(shs, want), (case, int((shs != want).sum()))


# ---- nsb_cage_set_membrane -----------------------------------------------------------------------------------------------------------
MIN_STEP = F64(1.73205080757 / 1024.0)


def _membrane_inputs(nv, n_cv, seed, with_nan):
    """gamma [nv, n_cv] with one-hot, all-zero, negative and tiny (subnormal product) rows; per cage vertex densities that are zero on
    one side, large enough for alpha = 1, subnormal on one side (alpha rounds to 0 in float32), ordinary, and with `with_nan` zero on
    both sides (0/0: w_inside NaN, which reaches every SH entry of every vertex); SH in both directions."""
    rng = np.random.default_rng(seed)
    g = rng.uniform(0.0, 1.0, (nv, n_cv)).astype(F32)
    g /= g.sum(1, keepdims=True)
    kinds = np.arange(nv) % 5
    g[kinds == 1] = 0.0
    g[kinds == 1, rng.integers(0, n_cv, int((kinds == 1).sum()))] = 1.0            # one-hot
    g[kinds == 2] = 0.0                                                            # all zero
    neg = kinds == 3
    g[neg] = rng.uniform(-0.4, 1.0, (int(neg.sum()), n_cv)).astype(F32)            # negative entries
    g[kinds == 4] *= F32(1e-37)                                                    # g * alpha subnormal
    d_in = rng.uniform(0.0, 60.0, n_cv).astype(F32)
    d_out = rng.uniform(0.0, 60.0, n_cv).astype(F32)
    k = np.arange(n_cv) % 7
    d_in[k == 1] = 0.0                                     # alpha_in = 0: w_inside 0
    d_out[k == 2] = 0.0                                    # alpha_out = 0: w_inside min(x / 0, 1) = 1
    if with_nan:
        d_in[k == 3] = d_out[k == 3] = 0.0                 # 0 / 0: w_inside NaN
    d_out[k == 4] = 1e5                                    # alpha_out = 1
    d_in[k == 5] = 1e-40                                   # subnormal densities: alpha 0 in float32, not in float64
    d_out[k == 6] = 3e-39
    s_in = rng.uniform(-1.0, 1.0, (n_cv, 27)).astype(F32)
    s_out = rng.uniform(-1.0, 1.0, (n_cv, 27)).astype(F32)
    return g, d_in, d_out, s_in, s_out


def _membrane_model(g, d_in, d_out, s_in, s_out):
    """interpolate_poisson_boundary (growing_selection.cu:2363-2392) in float64, and a bound on the float32 evaluation's distance to it:
    alpha = 1 - expf(-d * step) is within 2^-23 absolute (libm expf within 1 ulp, the subtraction within one rounding); w_inside =
    min(alpha_in / alpha_out, 1) is within its relative perturbation; each of the n_cv-term sums within gamma_{n+3} of its sum of |terms|;
    then the quotient's first-order error and a final rounding. Every rounding of a subnormal adds up to 2^-150 absolute: (n + 3) 2^-149
    covers a sum's."""
    ea = 2.0 ** -23
    g, d_in, d_out, s_in, s_out = (x.astype(F64) for x in (g, d_in, d_out, s_in, s_out))
    a_out, a_in = -np.expm1(-d_out * F64(F32(MIN_STEP))), -np.expm1(-d_in * F64(F32(MIN_STEP)))
    ea_out, ea_in = np.where(d_out == 0, 0.0, ea), np.where(d_in == 0, 0.0, ea)  # a zero density gives alpha exactly 0
    with np.errstate(divide="ignore", invalid="ignore"):
        q = a_in / a_out
        w = np.minimum(q, 1.0)
        dw = np.where(q < 1.0, q * (ea_in / np.maximum(a_in, 1e-300) + ea_out / np.maximum(a_out, 1e-300) + U), 0.0)
        dw = np.where(np.isfinite(dw), np.minimum(dw, 2.0), 2.0)                     # w stays in [0, 1]
    D = s_out[None] - w[:, None] * s_in                                                # [n_cv, 27]
    dD = dw[:, None] * np.abs(s_in) + 2 * U * (np.abs(s_out) + np.abs(w[:, None] * s_in))
    ga = g * a_out[None]
    num = ga @ D
    den = ga.sum(1) + 1e-6
    n = g.shape[1]
    gam = (n + 3) * U / (1 - (n + 3) * U)
    sub = (n + 3) * 2.0 ** -149
    dnum = np.abs(g) @ (ea_out[:, None] * np.abs(D) + a_out[:, None] * dD) + (gam + 2 * U) * (np.abs(ga) @ np.abs(D)) + sub
    dden = np.abs(g) @ ea_out + (gam + 2 * U) * np.abs(ga).sum(1) + U * 1e-6 + sub
    sh = num / den[:, None]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        dsh = dnum / np.abs(den)[:, None] + np.abs(num) * dden[:, None] / (den ** 2)[:, None] + U * np.abs(sh) + 1e-45
    od = g @ d_out
    dod = gam * (np.abs(g) @ np.abs(d_out)) + sub
    rd = g @ (d_out - d_in)
    drd = (gam + U) * (np.abs(g) @ np.abs(d_out - d_in)) + sub  # d_out - d_in rounded once
    return (sh, dsh), (od, dod), (np.maximum(rd, 0.0), drd)


# (lattice cells per side, [n_cv, ...]): nv = (cells + 1)^3 = 8, 27, 64, 2197; several n_cv in turn re-blend the same operator
BLEND_CASES = {"cells1": (1, [4, 26]), "cells2": (2, [386, 4]), "cells3": (3, [26, 386, 26]), "cells12": (12, [26, 4, 386])}


@pytest.mark.parametrize("case", list(BLEND_CASES))
def test_cage_set_membrane_domain(scene, renderer, case):
    """k_membrane_blend on lattice cages whose vertex counts leave a partial CTA, re-blended with other n_cv: bit for bit against
    oracle.membrane_blend (NaN equal to NaN: the 0/0 path of w_inside), and every non-NaN entry within the float64 model's bound."""
    model, _ = scene
    cells, ncvs = BLEND_CASES[case]
    op = fx.make_cage(model, (0.5, 0.62, 0.78), (0.17, 0.17, 0.17), n_lattice=cells)
    nv = op.vertices.shape[0]
    assert nv == (cells + 1) ** 3
    worst = 0.0
    n_nan = 0
    try:
        renderer.set_edit_operators([op.to_op()])
        for k, n_cv in enumerate(ncvs):
            g, d_in, d_out, s_in, s_out = _membrane_inputs(nv, n_cv, seed=100 * cells + k, with_nan=k > 0)
            b_shs, b_od, b_rd = renderer.cage_set_membrane(0, g, d_in, d_out, s_in, s_out, amplitude=1.0, apply=True)
            o_shs, o_od, o_rd = orc.membrane_blend(g, d_in, d_out, s_in, s_out)
            assert _same(b_shs, o_shs), (case, n_cv, int((~((b_shs == o_shs) | (np.isnan(b_shs) & np.isnan(o_shs)))).sum()))
            assert _same(b_od, o_od) and _same(b_rd, o_rd), (case, n_cv)
            assert np.isnan(b_shs).all() if k > 0 else not np.isnan(b_shs).any(), "the 0/0 path of w_inside reaches every SH entry"
            n_nan += int(np.isnan(b_shs).sum())
            for got, (m, bound) in zip((b_shs, b_od, b_rd), _membrane_model(g, d_in, d_out, s_in, s_out)):
                ok = ~np.isnan(got) & np.isfinite(m) & np.isfinite(bound)
                if not ok.any():  # the 0/0 path: every SH entry is NaN
                    continue
                err = np.abs(got.astype(F64) - m)
                assert (err[ok] <= bound[ok]).all(), (case, n_cv, float((err / bound)[ok].max()))
                worst = max(worst, float((err / bound)[ok].max()))
    finally:
        renderer.reset_edit_operators()
    print(f"\nmembrane blend {case}: nv {nv} ({(nv + 3) // 4} CTAs), n_cv {ncvs}: bit for bit ({n_nan} NaN entries); float64 model "
          f"largest err/bound {worst:.3f}")
