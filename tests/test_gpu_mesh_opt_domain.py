"""Mesh optimisation on the H100 over its whole domain (inputs: tests/mesh_opt_domain.py), under both MLP accumulator policies.

* nsb_density_gradient on every grid geometry, at every position class (out of the cube, lattice points of the dense levels, inf / NaN)
  and a ragged row count: the raw density is nsb_density's bit for bit (padded rows included), dfeat meets the MLP contract against the
  oracle, and the grid backward of the device's own dfeat is the oracle's bit for bit (NaN compared as a class).
* Several tiles per CTA: one call over four waves and more equals the concatenation of calls of less than a wave each, and late tiles
  equal the oracle; one nsb_mesh_optimise step on a mesh of more than 2^20 rows equals the CPU mirror.
* One step on every mesh x parameter row x train AABB equals the mirror; 300 chained steps (the amounts switched halfway) equal the mirror
  step by step, with the mirror's own Adam state and the device's debiasing powers, and two calls on a fresh context land on the same bytes.
* Optimiser state lifetime: a shade between two calls, an odd step count before a re-mesh to a larger mesh, a side stream; an empty mesh.
* The reference's own opt gradient (oracle/_ref, replayed from tests/golden/ref/ where it is absent) on a table of the cases above.
"""
import ctypes as C

import numpy as np
import pytest

import encoding_domain as ed
import mesh_opt_domain as mod
import ref_golden as rg
from nerfshop_b200 import abi
from oracle import ref_mesh_opt, ref_mesh_opt_build
from test_gpu_density_gradient import _ulps
from test_gpu_mesh_optimise import _download
from test_gpu_mesh_optimise_ref import agree_with_reference

pytestmark = pytest.mark.gpu

POLICIES = {"f32": (abi.NSB_MLP_ACC_F32, 0), "f16": (abi.NSB_MLP_ACC_F16, 1)}  # device policy, oracle policy
GRAD_SMEM_MIN = 20480 + 8192 + 4096  # meshopt::GradSmem: the MLP weights, the tile's operand space and W1^T, at least


def _torch():
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _renderer(desc, params, density_grid=None):
    _torch()
    from nerfshop_b200.renderer import NerfRenderer

    r = NerfRenderer(0)
    r.upload_model(desc, params)
    if density_grid is not None:
        r.upload_density_grid(density_grid)
    return r


def _fox_renderer(scene):
    model, occ = scene
    return _renderer(model.desc, model.params, np.unpackbits(occ, bitorder="little").astype(np.float32))


@pytest.fixture(scope="module")
def fr(scene, built_lib):
    r = _fox_renderer(scene)
    yield r
    r.close()


@pytest.fixture(scope="module")
def pows():
    _torch()
    p = mod.device_pows(4096)
    h = mod.host_pows(4096)
    for n in (301, 1001, 4096):
        print(f"\npowf(0.9f, t), powf(0.99f, t) for t = 1..{n - 1}: the device's and the host's differ at {(p[1:n, 0] != h[1:n, 0]).sum()} and "
              f"{(p[1:n, 1] != h[1:n, 1]).sum()} values of t")
    return p


def _waves(torch):
    """(SMs, the most CTAs of nsb_density_gradient the shared memory lets one SM hold)."""
    props = torch.cuda.get_device_properties(0)
    return props.multi_processor_count, props.shared_memory_per_multiprocessor // (GRAD_SMEM_MIN + 1024)


# ---- the meshes, on the device -------------------------------------------------------------------------------------------------
_grids = {}


def _source(r, source, res):
    """(density grid on the device, res, (box min, box max), threshold)."""
    torch = _torch()
    key = (source, res)
    if key not in _grids:
        if source == "fox":
            d = r.density_on_grid((res, res, res), mod.md.FOX, mod.md.FOX)
            v = d.cpu().numpy().reshape(-1)
            _grids[key] = (d, (res, res, res), mod.md.FOX, float(np.median(v[v > -10000.0])))
        else:
            f, box, t = mod.field(source)
            rz, ry, rx = f.shape
            _grids[key] = (torch.as_tensor(f).cuda(), (rx, ry, rz), box, t)
    return _grids[key]


def _remesh(r, spec, stream=None):
    """Meshes `spec` (a MESHES row) in r: (n_vertices, n_indices, threshold)."""
    source, res, _ = spec
    d, res3, box, t = _source(r, source, res)
    nv, ni = r.marching_cubes(d, res3, box, t, stream=stream)
    return nv, ni, t


def _step_vs_mirror(r, nv, ni, thresh, train, k, pows, state=None):
    """One nsb_mesh_optimise step against the mirror fed the device's density and gradient at the same rows: (V1, state)."""
    from oracle import mesh_opt_oracle as mo

    V0, _, F0 = _download(r, nv, ni, normals=False)
    grad, dens = r.density_gradient(mod.warp(V0, train))
    r.mesh_optimise(1, thresh, train, *k)
    V1, N1, F1 = _download(r, nv, ni)
    np.testing.assert_array_equal(F1, F0)
    P, N, state = mo.mesh_opt_step(V0, F0, dens, grad, thresh, *k, state, pows=pows)
    bad_n, bad_v = ~mod.same_or_both_nan(N1, N), ~mod.same_or_both_nan(V1, P)
    assert not bad_n.any(), f"normals differ on {bad_n.any(1).sum()} rows, first {np.argwhere(bad_n)[:4].tolist()}"
    assert not bad_v.any(), f"positions differ on {bad_v.any(1).sum()} rows, first {np.argwhere(bad_v)[:4].tolist()}"
    return V0, V1, dens, state


# ---- 1. nsb_density_gradient on every geometry ------------------------------------------------------------------------------
def _gradient_raw(r, coords, sentinel=0x7BCD):
    """nsb_density_gradient's full outputs: grad [n, 3], density fp16 bits [n_padded], dfeat fp16 bits [32, n_padded]."""
    torch = _torch()
    c = torch.as_tensor(np.ascontiguousarray(coords, np.float32)).cuda()
    n = c.shape[0]
    n_pad = (n + 127) // 128 * 128
    g = torch.zeros((n, 3), dtype=torch.float32, device="cuda")
    d = torch.full((n_pad,), sentinel, dtype=torch.int16, device="cuda")
    df = torch.full((32, n_pad), sentinel, dtype=torch.int16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    assert r.lib.nsb_density_gradient(r.ctx, c.data_ptr(), n, g.data_ptr(), 3, d.data_ptr(), df.data_ptr(), n_pad, st) == 0, r.lib.nsb_last_error()
    torch.cuda.synchronize()
    return g.cpu().numpy(), d.cpu().numpy().view(np.uint16), df.cpu().numpy().view(np.uint16)


def _density_raw(r, coords):
    """nsb_density's density row over all n_padded rows."""
    torch = _torch()
    c = torch.as_tensor(np.ascontiguousarray(coords, np.float32)).cuda()
    n = c.shape[0]
    n_pad = (n + 127) // 128 * 128
    out = torch.full((16, n_pad), 0x3C01, dtype=torch.int16, device="cuda")
    assert r.lib.nsb_density(r.ctx, c.data_ptr(), n, out.data_ptr(), n_pad, torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()
    return out.cpu().numpy().view(np.uint16)[0]


def _check_against_oracle(o, coords, grad, dfeat, what):
    """dfeat within the MLP contract of the oracle's (NaN as a class), the grid backward of the device's dfeat bit for bit."""
    from oracle import mesh_opt_oracle as mo

    _, df_o, _ = mo.density_gradient(o, coords)
    g_given, _, _ = mo.density_gradient(o, coords, dfeat=dfeat)
    nan_d, nan_o = np.isnan(dfeat.view(np.float16)), np.isnan(df_o.view(np.float16))
    assert (nan_d == nan_o).all(), f"{what}: dfeat NaN on {(nan_d != nan_o).sum()} other halves"
    u = _ulps(dfeat[~nan_d], df_o[~nan_o])
    eq = (u == 0).mean()
    print(f"\n{what}: dfeat {100 * eq:.3f} % bit-equal, max {u.max()} ulp over {dfeat.size} halves ({nan_d.sum()} NaN)")
    assert eq >= 0.999 and u.max() <= 4, (eq, u.max())
    bad = ~mod.same_or_both_nan(grad, g_given)
    assert not bad.any(), f"{what}: grid backward differs on {bad.any(1).sum()} rows, first {np.argwhere(bad)[:4].tolist()}"
    return eq


@pytest.mark.parametrize("policy", sorted(POLICIES))
@pytest.mark.parametrize("name", list(ed.GEOMETRIES))
def test_density_gradient_on_every_geometry(built_lib, name, policy):
    from oracle import mesh_opt_oracle as mo
    from oracle import oracle as orc

    d = ed.GEOMETRIES[name]
    params = ed.make_model(d, seed=5)
    coords = ed.coord_rows(ed.positions(*ed.level_geometry(d)), seed=4, specials=True)
    coords = coords[: coords.shape[0] - (1 if coords.shape[0] % 128 == 0 else 0)]
    n = coords.shape[0]
    assert n % 128 != 0 and (~np.isfinite(coords[:, :3])).any(1).sum() > 0
    dev_policy, orc_policy = POLICIES[policy]
    r = _renderer(d, params)
    old = mo.set_mlp_policy(orc_policy)
    try:
        r.set_mlp_accumulator(dev_policy)
        grad, dens, dfeat = _gradient_raw(r, coords)
        raw = _density_raw(r, coords)
        np.testing.assert_array_equal(dens, raw)  # nsb_density's, padded rows included
        assert (dens != 0x7BCD).all() and (dfeat != 0x7BCD).any(0).all()  # every padded row written
        _check_against_oracle(orc.Oracle(d, params, None), coords, grad, dfeat[:, :n], f"{name} {policy}")
    finally:
        mo.set_mlp_policy(old)
        r.close()
    assert np.isnan(grad).any() and np.isfinite(grad).all(1).mean() > 0.5


# ---- 2. several tiles per CTA ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("policy", sorted(POLICIES))
def test_density_gradient_over_several_tiles_per_cta(fr, scene, oracle, policy):
    from conftest import random_coords
    from oracle import mesh_opt_oracle as mo

    torch = _torch()
    sms, cps = _waves(torch)
    wave = sms * cps * 128
    n = 4 * wave + 77
    coords = random_coords(n, seed=8)
    extra = ed.coord_rows(ed.positions(*ed.level_geometry(scene[0].desc)), seed=6, specials=True)
    coords[-extra.shape[0]:] = extra  # the position classes, in the last tiles
    dev_policy, orc_policy = POLICIES[policy]
    fr.set_mlp_accumulator(dev_policy)
    old = mo.set_mlp_policy(orc_policy)
    try:
        g, d, df = _gradient_raw(fr, coords)
        chunk = sms * 128  # one tile per CTA at any residency
        parts = [_gradient_raw(fr, coords[a:a + chunk]) for a in range(0, n, chunk)]
        np.testing.assert_array_equal(g.view(np.uint32), np.concatenate([p[0] for p in parts]).view(np.uint32))
        np.testing.assert_array_equal(d[:n], np.concatenate([p[1][: min(chunk, n - i * chunk)] for i, p in enumerate(parts)]))
        np.testing.assert_array_equal(df[:, :n], np.concatenate([p[2][:, : min(chunk, n - i * chunk)] for i, p in enumerate(parts)], 1))
        late = np.sort(np.random.default_rng(2).choice(np.arange(3 * wave, n), 4096, replace=False))
        late = np.union1d(late, np.arange(n - extra.shape[0], n))
        _check_against_oracle(oracle, coords[late], g[late], df[:, late], f"tiles past the third wave ({sms} SMs x {cps} CTAs), {policy}")
    finally:
        mo.set_mlp_policy(old)
        fr.set_mlp_accumulator(abi.NSB_MLP_ACC_F16)


@pytest.mark.parametrize("policy", sorted(POLICIES))
def test_one_step_on_a_mesh_of_several_waves(fr, pows, policy):
    torch = _torch()
    sms, cps = _waves(torch)
    fr.set_mlp_accumulator(POLICIES[policy][0])
    try:
        nv, ni, t = _remesh(fr, mod.BIG)
        rows = (nv + 127) // 128 * 128
        print(f"\n{nv} vertices, {rows // 128} tiles = {rows / (128 * sms * cps):.1f} waves of {sms} x {cps} CTAs")
        assert rows >= 1 << 20 and rows // 128 >= 4 * sms * cps
        V0, V1, _, _ = _step_vs_mirror(fr, nv, ni, t, mod.TRAINS["fox"], (2048.0, 128.0, 1.0), pows)
        assert (V1 != V0).mean() > 0.9
    finally:
        fr.set_mlp_accumulator(abi.NSB_MLP_ACC_F16)


# ---- 3. one step on every mesh x parameter row x train AABB -----------------------------------------------------------------
@pytest.mark.parametrize("policy", sorted(POLICIES))
@pytest.mark.parametrize("mesh", list(mod.MESHES))
def test_one_step_on_every_case_equals_the_mirror(fr, pows, mesh, policy):
    spec = mod.MESHES[mesh]
    fr.set_mlp_accumulator(POLICIES[policy][0])
    try:
        nv, ni, t_mesh = _remesh(fr, spec)
        rows = (nv + 127) // 128 * 128
        assert nv > 0 and (mesh != "octahedra_384" or nv == rows == 384)
        moved = {}
        for train_name, train in mod.TRAINS.items():
            for pname, (tk, *k) in mod.PARAMS.items():
                nv, ni, _ = _remesh(fr, spec)  # a fresh optimiser
                thresh = t_mesh
                if tk == "vertex":
                    V, _, _ = _download(fr, nv, ni, normals=False)
                    thresh = mod.thresh_of(tk, t_mesh, fr.density_gradient(mod.warp(V, train))[1], nv)
                elif tk != "mesh":
                    thresh = float(tk)
                V0, V1, _, _ = _step_vs_mirror(fr, nv, ni, thresh, train, tuple(k), pows)
                fin = np.isfinite(V0).all(1)
                moved[(train_name, pname)] = (V1[fin] != V0[fin]).mean() if fin.all() else (~mod.same_or_both_nan(V1, V0)).mean()
        if mesh != "inf_nan_and_filter_value":  # an infinite 1-ring sum times an amount of 0 is NaN, a gradient that steps
            assert all(moved[(tn, "all_zero")] == 0 for tn in mod.TRAINS)
        print(f"\n{mesh} ({nv} vertices) {policy}: share of coordinates moved per case: " + ", ".join(f"{a}/{b} {v:.2f}" for (a, b), v in moved.items()))
    finally:
        fr.set_mlp_accumulator(abi.NSB_MLP_ACC_F16)


# ---- 4. many steps, chained ---------------------------------------------------------------------------------------------------
CHAINS = {  # mesh -> (first amounts, second amounts): smooth (or inflate) only, then density only
    "fox_train_non_pow2": ((2048.0, 0.0, 0.0), (0.0, 128.0, 0.0)),
    "box_zero_extent_y": ((0.0, 0.0, 1.0), (0.0, 128.0, 0.0)),  # normals along y only: x and z start stepping with the density term
}
N_CHAIN = 300


@pytest.mark.parametrize("policy", sorted(POLICIES))
@pytest.mark.parametrize("mesh", list(CHAINS))
def test_many_steps_equal_the_mirror_step_by_step(fr, scene, pows, mesh, policy):
    spec = mod.MESHES[mesh]
    train = mod.TRAINS[spec[2]]
    k1, k2 = CHAINS[mesh]
    fr.set_mlp_accumulator(POLICIES[policy][0])
    fresh = _fox_renderer(scene)
    try:
        nv, ni, t = _remesh(fr, spec)
        rows = (nv + 127) // 128 * 128
        assert rows > nv  # padding rows at the origin
        state = None
        for s in range(N_CHAIN):
            k = k1 if s < N_CHAIN // 2 else k2
            _, V1, _, state = _step_vs_mirror(fr, nv, ni, t, train, k, pows, state)
            steps = state[2]
            if s == N_CHAIN // 2 - 1:
                assert (steps[nv:] == 0).all()  # the padding sat at its centroid: no step yet
            if s == N_CHAIN // 2:
                assert (steps[nv:] == 1).all()  # their first density step is debiased as t = 1
                assert (steps[:nv] > 1).any()
        assert steps.max() > N_CHAIN // 2 and len(np.unique(steps)) > 2
        print(f"\n{mesh} {policy}: {N_CHAIN} steps bit for bit; per-coordinate step counts {np.unique(steps).tolist()[:8]}...")
        # the same 300 steps in two calls on a fresh context
        fresh.set_mlp_accumulator(POLICIES[policy][0])
        nvf, nif, _ = _remesh(fresh, spec)
        fresh.mesh_optimise(N_CHAIN // 2, t, train, *k1)
        fresh.mesh_optimise(N_CHAIN - N_CHAIN // 2, t, train, *k2)
        Vf, Nf, _ = _download(fresh, nvf, nif)
        V, N, _ = _download(fr, nv, ni)
        assert Vf.tobytes() == V.tobytes() and Nf.tobytes() == N.tobytes()
    finally:
        fresh.close()
        fr.set_mlp_accumulator(abi.NSB_MLP_ACC_F16)


# ---- 5. optimiser state lifetime ------------------------------------------------------------------------------------------------
def test_a_shade_between_calls_changes_nothing(fr, scene):
    spec, train = mod.MESHES["fox"], mod.TRAINS["fox"]
    nv, ni, t = _remesh(fr, spec)
    fr.mesh_optimise(3, t, train)
    fr.mesh_shade(train)
    fr.mesh_optimise(3, t, train)
    V, N, _ = _download(fr, nv, ni)
    other = _fox_renderer(scene)
    try:
        _remesh(other, spec)
        other.mesh_optimise(6, t, train)
        Vo, No, _ = _download(other, nv, ni)
    finally:
        other.close()
    assert V.tobytes() == Vo.tobytes() and N.tobytes() == No.tobytes()


def test_odd_steps_then_a_larger_mesh_equals_a_fresh_context(fr, scene):
    small, large = ("fox", 32, "fox"), mod.MESHES["fox_train_non_pow2"]
    train = mod.TRAINS["non_pow2"]
    nv0, _, t0 = _remesh(fr, small)
    fr.mesh_optimise(7, t0, train)  # odd: the mesh now lives in the second ping-pong buffer
    nv, ni, t = _remesh(fr, large)
    assert nv > 2 * nv0
    fr.mesh_optimise(5, t, train)
    V, N, F = _download(fr, nv, ni)
    other = _fox_renderer(scene)
    try:
        _remesh(other, large)
        other.mesh_optimise(5, t, train)
        Vo, No, Fo = _download(other, nv, ni)
    finally:
        other.close()
    assert V.tobytes() == Vo.tobytes() and N.tobytes() == No.tobytes() and F.tobytes() == Fo.tobytes()


def test_side_stream_equals_the_default_stream(fr, scene):
    torch = _torch()
    spec, train = mod.MESHES["fox_partly_outside"], mod.TRAINS["unit"]
    nv, ni, t = _remesh(fr, spec)
    fr.mesh_optimise(9, t, train)
    V, N, _ = _download(fr, nv, ni)
    other = _fox_renderer(scene)
    try:
        s = torch.cuda.Stream()
        _source(other, spec[0], spec[1])
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            _remesh(other, spec, stream=s.cuda_stream)
            other.mesh_optimise(9, t, train, stream=s.cuda_stream)
        s.synchronize()
        Vo, No, _ = _download(other, nv, ni)
    finally:
        other.close()
    assert V.tobytes() == Vo.tobytes() and N.tobytes() == No.tobytes()


@pytest.mark.parametrize("first", ["optimise", "shade"])
def test_empty_mesh_has_normals_after_either_call(fr, first):
    """An empty mesh has no normals to compute: nsb_mesh_optimise and nsb_mesh_shade both leave it with (empty) normals, in either order."""
    nv, ni, t = _remesh(fr, ("all_outside", None, "fox"))
    assert nv == ni == 0
    train = mod.TRAINS["fox"]
    V = np.zeros((1, 3), np.float32)
    calls = [lambda: fr.mesh_optimise(1, t, train), lambda: fr.mesh_shade(train)]
    for call in (calls if first == "optimise" else calls[::-1]):
        call()
        assert fr.lib.nsb_mesh_download(fr.ctx, None, V.ctypes.data, None, 0, None, 0) == abi.NSB_OK, fr.lib.nsb_last_error()
    assert fr.lib.nsb_mesh_download(fr.ctx, V.ctypes.data, V.ctypes.data, V.ctypes.data, 0, None, 0) == abi.NSB_OK


# ---- 6. the reference's opt gradient --------------------------------------------------------------------------------------------
HAVE = ref_mesh_opt_build.build() is not None
REF_CASES = {  # name -> (mesh, parameter row, train AABB); the least share of rows whose atomic sums agree, measured below
    "non_pow2_train": ("fox_train_non_pow2", "reference", "non_pow2"),
    "partly_outside": ("fox_partly_outside", "reference", "unit"),
    "all_zero": ("fox", "all_zero", "fox"),
    "smooth_only": ("fox", "smooth_only", "fox"),
    "density_only": ("fox", "density_only", "fox"),
    "inflate_only": ("fox", "inflate_only", "fox"),
    "thresh_at_vertex": ("fox", "thresh_at_vertex", "fox"),
    "thresh_pos_nan": ("fox", "thresh_pos_nan", "fox"),
    "thresh_neg_nan": ("fox", "thresh_neg_nan", "fox"),
    "checkerboard": ("checkerboard", "reference", "non_pow2"),
}


@pytest.mark.skipif(not (HAVE or rg._stored("test_gpu_mesh_opt_domain")), reason="neither oracle/_ref nor stored reference results (tests/golden/ref/)")
@pytest.mark.parametrize("case", list(REF_CASES))
def test_opt_gradient_vs_reference(fr, case):
    from oracle import mesh_opt_oracle as mo

    mesh, pname, train_name = REF_CASES[case]
    train = mod.TRAINS[train_name]
    tk, *k = mod.PARAMS[pname]
    nv, ni, t_mesh = _remesh(fr, mod.MESHES[mesh])
    V0, _, F = _download(fr, nv, ni, normals=False)
    grad, dens = fr.density_gradient(mod.warp(V0, train))
    thresh = t_mesh if tk == "mesh" else mod.thresh_of(tk, t_mesh, dens, nv) if tk == "vertex" else float(tk)
    g7 = np.zeros((V0.shape[0], 7), np.float32)  # the reference reads the gradient in place of its network inputs (stride 7)
    g7[:, :3] = grad
    g_ref, s_ref, n_ref = rg._call(HAVE, ref_mesh_opt.opt_gradients if HAVE else None, V0, F, dens, g7, thresh, *k)
    rows = np.asarray(g_ref.rows) if isinstance(g_ref, rg.Sampled) else np.arange(V0.shape[0])
    g_ref, s_ref, n_ref = (np.asarray(a).view(np.ndarray) for a in (g_ref, s_ref, n_ref))
    s_our, n_our, g_our = (a[rows] for a in mo.mesh_opt_gradient(V0, F, dens, grad, thresh, *k))
    fr.mesh_optimise(1, thresh, train, *k)
    V1 = _download(fr, nv, ni, normals=False)[0][rows]
    P_ref, _ = mo.adam_step(V0[rows], g_ref)
    share = agree_with_reference(rows, nv, V1, P_ref, g_our, g_ref, s_our, s_ref, n_our, n_ref, min_agree=0.3)
    print(f"{case}: {100 * share:.2f} % of the rows agree with the reference bit for bit")
    if pname == "all_zero":
        assert (V1 == V0[rows]).all()
