"""The hash-grid encoding on the H100 over its whole input domain: positions outside [0,1]^3 (down to +-1e6, where the float->int
conversion saturates, and +-inf / NaN), and a table of level geometries (tests/encoding_domain.py), against the CPU oracle.

Bars as in test_gpu_parity.py / test_gpu_density_gradient.py: the encoding bit for bit (NaN features compared as NaN), MLP outputs within
the fp16 ulp bars, frames within _compare_frames. The grid index is pinned on the CPU first: test_encoding_domain_cpu.py runs the
product's grid_index on every grid coordinate the position classes below reach, on each axis against structured partners, plus random
uint32 triples. Then edit operators whose geometry leaves the train AABB (render and grid update), and mesh shading and optimisation
against a train AABB that leaves part of the mesh and the padding rows outside."""
import numpy as np
import pytest

import encoding_domain as ed
from nerfshop_b200 import abi, synthetic as syn
from test_gpu_parity import _compare_frames, _half, _ulp_close

pytestmark = pytest.mark.gpu

FOX_TRAIN = ((-1.5, -1.5, -1.5), (2.5, 2.5, 2.5))
POLICIES = {"f32": (abi.NSB_MLP_ACC_F32, 0), "f16": (abi.NSB_MLP_ACC_F16, 1)}  # device policy, oracle policy


def _renderer(d, params, occ=None):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nerfshop_b200.renderer import NerfRenderer

    r = NerfRenderer(0)
    r.upload_model(d, params)
    if occ is not None:
        r.upload_occupancy(occ)
    return r


def _out_of_cube_rows(d, specials=False, seed=2):
    return ed.coord_rows(ed.positions(*ed.level_geometry(d)), seed=seed, specials=specials)


@pytest.mark.parametrize("name", list(ed.GEOMETRIES))
def test_encode_bit_exact_on_the_whole_domain(built_lib, name):
    from oracle import oracle as orc

    d = ed.GEOMETRIES[name]
    params = ed.make_model(d, seed=5)
    rows = _out_of_cube_rows(d, specials=True)
    ref = orc.Oracle(d, params, None).encode(rows)
    r = _renderer(d, params)
    try:
        got = r.encode(rows)
    finally:
        r.close()
    nan_g, nan_r = np.isnan(got.view(np.float16)), np.isnan(ref.view(np.float16))
    assert (nan_g == nan_r).all(), f"{name}: NaN features differ on {(nan_g != nan_r).sum()} halves"
    assert (got[~nan_g] == ref[~nan_r]).all(), f"{name}: {(got[~nan_g] != ref[~nan_r]).sum()} of {got.size} fp16 features differ"
    assert (~np.isfinite(rows[:, :3]).all(1)).sum() > 0 and nan_g.any()


@pytest.mark.parametrize("policy", sorted(POLICIES))
def test_density_and_inference_out_of_the_cube(scene, built_lib, policy):
    from oracle import oracle as orc

    model, _ = scene
    dev_policy, orc_policy = POLICIES[policy]
    rows = _out_of_cube_rows(model.desc)
    outside = ((rows[:, :3] < 0) | (rows[:, :3] > 1)).any(1)
    assert outside.mean() > 0.5
    o = orc.Oracle(model.desc, model.params, None)
    old = orc.set_mlp_policy(orc_policy)
    r = _renderer(model.desc, model.params)
    try:
        r.set_mlp_accumulator(dev_policy)
        got_d, got = r.density(rows), r.inference(rows)
        ref_d, ref = o.inference(rows, density_only=True), o.inference(rows)
    finally:
        orc.set_mlp_policy(old)
        r.close()
    bad = _ulp_close(got_d, ref_d)
    assert bad.mean() < 1e-3, f"density MLP: {bad.sum()} of {bad.size} outputs off by more than 2 ulp"
    assert (got[3] == got_d[0]).all()
    bad = _ulp_close(got[:4], ref[:4], ulps=4, atol=2e-3)
    assert bad.mean() < 2e-3, f"rgb MLP: {bad.sum()} of {bad.size} outputs outside tolerance"
    assert np.abs(_half(got[:3]) - _half(ref[:3])).max() < 0.05


@pytest.mark.parametrize("policy", sorted(POLICIES))
def test_density_gradient_out_of_the_cube(scene, oracle, built_lib, policy):
    from oracle import mesh_opt_oracle as mo
    from test_gpu_density_gradient import _ulps

    model, _ = scene
    dev_policy, orc_policy = POLICIES[policy]
    rows = _out_of_cube_rows(model.desc, seed=3)
    assert rows.shape[0] % 128 != 0
    r = _renderer(model.desc, model.params)
    old = mo.set_mlp_policy(orc_policy)
    try:
        r.set_mlp_accumulator(dev_policy)
        grad, dens, dfeat = r.density_gradient(rows, want_dfeat=True)
        raw = r.density(rows)[0]
        _, df_o, _ = mo.density_gradient(oracle, rows)
        g_given, _, _ = mo.density_gradient(oracle, rows, dfeat=dfeat)
    finally:
        mo.set_mlp_policy(old)
        r.close()
    np.testing.assert_array_equal(dens, raw)
    u = _ulps(dfeat, df_o)
    assert (u == 0).mean() >= 0.999 and u.max() <= 4, f"dfeat: {(u == 0).mean():.4f} bit-equal, max {u.max()} ulp"
    np.testing.assert_array_equal(grad.view(np.uint32), g_given.view(np.uint32))


def test_density_on_grid_past_the_train_aabb(scene, built_lib):
    """The box [-2.5, 5.5]^3 extends past the fox train AABB [-1.5, 2.5]^3 on every face (warped coordinates -0.25 .. 1.75). Extent 8 and
    res 64 are powers of two, so the grid positions and their warped coordinates are exact. The running density grid is all ones: no cell is
    filtered, so every point equals nsb_density at the same warped coordinates."""
    model, _ = scene
    res = 64
    box = ((-2.5, -2.5, -2.5), (5.5, 5.5, 5.5))
    r = _renderer(model.desc, model.params)
    try:
        r.upload_density_grid(np.ones(abi.NSB_NERF_CASCADES * abi.NSB_NERF_GRIDSIZE ** 3, np.float32))
        got = r.density_on_grid((res, res, res), box, FOX_TRAIN).cpu().numpy().reshape(-1)
        i = np.arange(res ** 3, dtype=np.int64)
        xyz = np.stack([i % res, (i // res) % res, i // (res * res)], 1).astype(np.float32)
        p = xyz * (np.float32(1.0) / np.float32(res)) * np.float32(8.0) + np.float32(-2.5)
        pw = (p - np.float32(-1.5)) / np.float32(4.0)
        assert (pw < 0).any() and (pw > 1).any()
        coords = np.zeros((pw.shape[0], 7), np.float32)
        coords[:, :3] = pw
        coords[:, 4:] = 0.5
        raw = r.density(coords)[0].view(np.float16).astype(np.float32)
    finally:
        r.close()
    np.testing.assert_array_equal(got.view(np.uint32), raw.view(np.uint32))


def _occupancy_with_outer_cascades(occ, seed=0, frac=0.02):
    """The scene's bitfield plus random bits in cascades 3 and 4, which cover space outside the fox train AABB."""
    bits = np.unpackbits(occ, bitorder="little").reshape(abi.NSB_NERF_CASCADES, -1)
    rng = np.random.default_rng(seed)
    for m in (3, 4):
        bits[m] |= rng.random(bits.shape[1]) < frac
    return np.packbits(bits.reshape(-1), bitorder="little")


def test_render_with_render_aabb_past_the_train_aabb(scene, built_lib):
    """Render AABB [-2.5, 3.5..4.5] around the fox train AABB [-1.5, 2.5]^3, occupancy in cascades 3-4 out there.
    For both cameras the march is bit-exact and the features of every marched sample (warped coordinates down to -0.25, up to 1.5) are the
    oracle's bit for bit. The frame is compared for the orbit camera. From above the scene (the second camera), a pixel whose opacity rests on
    three dense samples outside the cube moves by 1.4e-3 when one raw density differs by 1 fp16 ulp (4.28125 vs 4.2851562, the MLP's
    summation order, within its 2-ulp contract). So only its march and encoding are pinned."""
    from oracle import oracle as orc

    model, occ = scene
    occ2 = _occupancy_with_outer_cascades(occ)
    o = orc.Oracle(model.desc, model.params, occ2)
    r = _renderer(model.desc, model.params, occ2)
    try:
        for k, cam in enumerate((syn.orbit_cameras(120)[10], syn.look_at((0.5, 4.0, 5.0)))):
            f = syn.make_frame(model, cam, 96, 54)
            for a in range(3):
                f.render_aabb_min[a], f.render_aabb_max[a] = -2.5, 3.5 + 0.5 * a
            pix = np.arange(0, 96 * 54, 3, dtype=np.uint32)
            rec_o, idx_o, cnt_o = o.march_trace(f, pix, 256)
            rec_g, idx_g, cnt_g = r.march_trace(f, pix, 256)
            assert (cnt_o == cnt_g).all() and (idx_o == idx_g).all() and (rec_o.view(np.uint32) == rec_g.view(np.uint32)).all()
            live = np.arange(256)[None, :] < cnt_o[:, None]
            pw = (rec_o[live][:, 2:5] - np.float32(-1.5)) / np.float32(4.0)  # the train extent 4 is a power of two: the warp is exact
            assert ((pw < 0) | (pw > 1)).any(1).sum() > 100
            c = np.zeros((pw.shape[0], 7), np.float32)
            c[:, :3] = pw
            c[:, 4:] = 0.5
            assert (r.encode(c) == o.encode(c)).all()
            if k == 0:
                fb_o, depth_o, st_o, margin = o.render(f, want_margin=True)
                fb, depth = r.render(f)
                _compare_frames(fb.cpu().numpy(), depth.cpu().numpy(), fb_o, depth_o, margin)
                assert r.stats().n_rays_alive == st_o.n_rays_alive
                assert st_o.n_samples > 1000
    finally:
        r.close()


@pytest.mark.parametrize("name", ["log2_12", "log2_3", "aabb16"])
def test_render_small_frame_on_table_geometries(scene, built_lib, name):
    """Frames of the fox scene's geometry on a model of another level table (odd-index mixed pair, all hashed, aabb_scale 16's levels),
    once with the render AABB equal to the train AABB and once past it."""
    from oracle import oracle as orc

    model, occ = scene
    d = ed.GEOMETRIES[name]
    params = ed.make_model(d, seed=9)
    occ2 = _occupancy_with_outer_cascades(occ, seed=1)
    o = orc.Oracle(d, params, occ2)
    r = _renderer(d, params, occ2)
    try:
        for grow in (0.0, 1.0):
            f = syn.make_frame(model, syn.orbit_cameras(120)[50], 64, 36)
            for a in range(3):
                f.render_aabb_min[a] -= grow
                f.render_aabb_max[a] += grow
            fb_o, depth_o, st_o, margin = o.render(f, want_margin=True)
            fb, depth = r.render(f)
            _compare_frames(fb.cpu().numpy(), depth.cpu().numpy(), fb_o, depth_o, margin)
    finally:
        r.close()


# ---- edit operators whose geometry leaves the train AABB ------------------------------------------------------------------------
def _outside_ops(model):
    """An affine duplication whose source box (warped z in [-0.03, 0.07], around the shell of the scene's dome) crosses the train AABB's
    z = min face, copied 0.3 inwards; and a cage around the dome at world z = -1.42 whose canonical tets reach z = -1.536, below the face
    at -1.5, with its +x face pulled along +z, so that deformed positions inside the AABB map back to canonical ones outside it."""
    from nerfshop_b200 import editing

    affine = editing.AffineDuplication((0.5, 0.425, 0.02), (0.1, 0.1, 0.1), (0.0, 0.0, 0.3))
    cage = editing.lattice_cage(model, (0.5, 0.2, -1.42), (0.12, 0.12, 0.12), pull=(0.0, 0.0, 0.08))
    return [affine.to_op(), cage.to_op()]


def _coords_around(model, center, half, n, seed):
    from conftest import random_coords

    rng = np.random.default_rng(seed)
    p = np.asarray(center, np.float32) + (rng.random((n, 3)).astype(np.float32) * 2 - 1) * np.asarray(half, np.float32)
    c = random_coords(n, seed)
    c[:, :3] = (p - model.aabb_min) / (model.aabb_max - model.aabb_min)
    return c


def test_operators_map_in_cube_samples_outside_it(scene, renderer):
    """The backward map of both operators sends samples from inside the cube to outside it, bit for bit like the oracle."""
    from oracle import oracle as orc

    model, occ = scene
    ops = _outside_ops(model)
    o = orc.Oracle(model.desc, model.params, occ, ops)
    renderer.set_edit_operators(ops)
    try:
        c = np.concatenate([_coords_around(model, (0.5, 0.2, -1.42), (0.13, 0.13, 0.08), 20000, 1),
                            _coords_around(model, (0.5, 0.2, -0.22), (0.25, 0.25, 0.25), 20000, 2)])
        ref, mref = o.map_rays(c)
        got, mgot = renderer.map_rays(c)
    finally:
        renderer.reset_edit_operators()
    assert np.array_equal(mref, mgot) and np.array_equal(ref.view(np.uint32), got.view(np.uint32))
    inside = ((c[:, :3] >= 0) & (c[:, :3] <= 1)).all(1)
    mapped_out = inside & ((ref[:, :3] < 0) | (ref[:, :3] > 1)).any(1)
    cage_rows = np.arange(c.shape[0]) < 20000
    assert (mapped_out & cage_rows).sum() > 100 and (mapped_out & ~cage_rows).sum() > 100


def test_render_with_operators_outside_the_train_aabb(scene, renderer):
    from oracle import oracle as orc

    model, occ = scene
    ops = _outside_ops(model)
    full = np.full(abi.NSB_BITFIELD_BYTES, 255, np.uint8)  # every cell occupied: the march reaches the destination box and the cage
    o = orc.Oracle(model.desc, model.params, full, ops)
    renderer.set_edit_operators(ops)
    renderer.upload_occupancy(full)
    try:
        for cam in (syn.look_at((1.3, 0.6, -0.3), target=(0.5, 0.25, -1.2)), syn.look_at((0.5, 0.22, 0.05), target=(0.5, 0.2, -1.3))):
            f = syn.make_frame(model, cam, 96, 54, apply_operators=True)
            fb_o, depth_o, st_o, margin = o.render(f, want_margin=True)
            fb, depth = renderer.render(f)
            st = renderer.stats()
            _compare_frames(fb.cpu().numpy(), depth.cpu().numpy(), fb_o, depth_o, margin)
            assert abs(int(st.n_samples) - int(st_o.n_samples)) <= max(20, st_o.n_samples // 2000)
            assert st_o.n_samples > 1000
    finally:
        renderer.reset_edit_operators()
        renderer.upload_occupancy(occ)


def test_grid_update_through_operators_outside_the_train_aabb(scene, renderer):
    from nerfshop_b200.rng import Pcg32
    from oracle import oracle as orc
    from test_grid_update_cpu import grid_params
    from test_gpu_grid_update import _compare

    model, occ = scene
    ops = _outside_ops(model)
    o = orc.Oracle(model.desc, model.params, occ, ops)
    renderer.set_edit_operators(ops)
    try:
        rng = Pcg32(7)
        n = 3 * 128 ** 3
        u = grid_params(n, 0, rng, n_cascades=3)  # cascade 2 covers the whole train AABB, the operators' boxes included
        g_cpu, b_cpu, mean = o.update_density_grid(u, np.zeros(abi.NSB_GRID_CELLS, np.float32))
        renderer.update_density_grid(rng.copy(), 0, n, 0, reset_grid=True, n_cascades=3)
        g_gpu, b_gpu = renderer.download_density_grid()
        _compare(g_gpu, b_gpu, g_cpu, b_cpu, mean)
        g_plain, _, _ = orc.Oracle(model.desc, model.params, occ).update_density_grid(u, np.zeros(abi.NSB_GRID_CELLS, np.float32))
        assert (g_plain != g_cpu).sum() > 100  # the operators did change the grid
    finally:
        renderer.reset_edit_operators()
        renderer.upload_occupancy(occ)


# ---- mesh shading and optimisation against a train AABB that leaves part of the mesh outside --------------------------------------
MESH_BOX = FOX_TRAIN
SHADE_TRAIN = ((0.5, 0.5, 0.5), (2.5, 2.5, 2.5))  # extent 2: the warp (v - 0.5) / 2 is one rounding, like the device's; the origin is outside


def _warp_shade(V):
    return (V - np.float32(0.5)) / np.float32(2.0)


@pytest.fixture()
def mesh_r(scene, built_lib):
    model, occ = scene
    r = _renderer(model.desc, model.params)
    r.upload_density_grid(np.unpackbits(occ, bitorder="little").astype(np.float32))
    res = 64
    d = r.density_on_grid((res, res, res), MESH_BOX, MESH_BOX)
    v = d.cpu().numpy().reshape(-1)
    t = float(np.median(v[v > -10000.0]))
    nv, ni = r.marching_cubes(d, (res, res, res), MESH_BOX, t)
    yield r, nv, ni, t
    r.close()


def test_mesh_colours_outside_the_train_aabb(mesh_r):
    r, nv, ni, _ = mesh_r
    r.mesh_shade(SHADE_TRAIN, 0)  # rgb activation None: colours are the raw fp16 outputs
    m = r.mesh_download(nv, ni)
    V, Cc = m["V"][:nv], m["C"][:nv]
    pw = _warp_shade(V)
    outside = ((pw < 0) | (pw > 1)).any(1)
    assert outside.mean() > 0.3 and (~outside).sum() > 100
    dd = V.astype(np.float64) - 0.5  # the direction is normalize(pos - 0.5), as in test_gpu_mesh.test_normals_and_colours
    n = np.sqrt((dd * dd).sum(1))
    dirs = np.where(n[:, None] > 0, dd / np.where(n > 0, n, 1)[:, None], dd).astype(np.float32)
    coords = np.zeros((nv, 7), np.float32)
    coords[:, :3] = pw
    coords[:, 4:] = (dirs + np.float32(1.0)) * np.float32(0.5)
    raw = r.inference(coords)[:3].view(np.float16).astype(np.float32).T
    same = (raw == Cc).all(1)
    assert same[outside].mean() > 0.99 and same.mean() > 0.99  # direction bits may differ in the last place (float64 vs the FMA form)
    assert np.abs(raw - Cc).max() < 2e-2


def test_mesh_optimise_step_outside_the_train_aabb_equals_the_mirror(mesh_r):
    from oracle import mesh_opt_oracle as mo
    from test_gpu_mesh_optimise import _download

    r, nv, ni, t = mesh_r
    V0, _, F0 = _download(r, nv, ni, normals=False)
    pw = _warp_shade(V0)
    outside = ((pw < 0) | (pw > 1)).any(1)
    assert outside[:nv].mean() > 0.3 and outside[nv:].all() and V0.shape[0] > nv  # padding rows sit at the origin, outside
    c = np.zeros((V0.shape[0], 7), np.float32)
    c[:, :3] = pw
    c[:, 4:] = 0.5
    grad, dens = r.density_gradient(c)
    r.mesh_optimise(1, t, SHADE_TRAIN)
    V1, N1, F1 = _download(r, nv, ni)
    np.testing.assert_array_equal(F1, F0)
    P, N, _ = mo.mesh_opt_step(V0, F0, dens, grad, t, 2048.0, 128.0, 1.0)
    np.testing.assert_array_equal(N1.view(np.uint32), N.view(np.uint32))
    np.testing.assert_array_equal(V1.view(np.uint32), P.view(np.uint32))
    assert (V1[nv:] != 0).any() and (V1 != V0).mean() > 0.9
