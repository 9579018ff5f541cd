"""Mesh extraction on the H100 over the domain of tests/mesh_domain.py, bit for bit against the exact oracle (tests/mesh_oracle.py) and the
reference's own kernels (oracle/_ref/libnerfshop_ref_mesh_cuda.so, or their stored results under tests/golden/ref/).

  * nsb_density_on_grid on every grid query, with each density grid and under both accumulator policies: every point against nsb_density at
    the oracle's grid point plus the oracle's filter, and the compared rows against the reference's grid_samples_half_to_float; one grid
    of 256 x 256 x 512 points on a seeded sample and its first and last 4096 points;
  * nsb_marching_cubes on every field: vertices and triangles in order, padding included, against the oracle; against the reference the
    vertex multiset and the cells' directed boundary cycles (its order comes from atomics, and its table triangulates some cycles
    differently);
  * nsb_mesh_shade: normals against mesh_oracle.normals bit for bit (NaNs equal); colours against the reference's colour inputs, nsb_inference
    and extract_srgb_with_activation for every rgb activation, with and without linear colours, under both policies;
  * empty meshes, one context reused over meshes of different sizes, and the 32-bit index guard on a 720^3 checkerboard.
"""
import contextlib

import numpy as np
import pytest

import mesh_domain as md
import mesh_oracle as mo
import ref_golden as rg
from nerfshop_b200 import abi, mesh
from oracle import ref_mesh, ref_mesh_build

HAVE = ref_mesh_build.build() is not None
pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not (HAVE or rg._stored("test_gpu_mesh_domain")),
                               reason="neither oracle/_ref nor stored reference results (tests/golden/ref/)")
POLICIES = {"f16": abi.NSB_MLP_ACC_F16, "f32": abi.NSB_MLP_ACC_F32}
ACTIVATIONS = (abi.NSB_ACT_NONE, abi.NSB_ACT_RELU, abi.NSB_ACT_LOGISTIC, abi.NSB_ACT_EXPONENTIAL)


def R(name, *args):
    """The reference's result (live, or its stored replay); never a row sample."""
    v = rg._call(HAVE, getattr(ref_mesh, name), *args)
    for a in v if isinstance(v, tuple) else (v,):
        assert not isinstance(a, rg.Sampled)
    return v


def _renderer(scene, grid):
    from nerfshop_b200.renderer import NerfRenderer

    r = NerfRenderer(0)
    r.upload_model(scene[0].desc, scene[0].params)
    r.upload_density_grid(grid)
    return r


@pytest.fixture(scope="module")
def grids(scene):
    return md.density_grids(scene[1])


@pytest.fixture(scope="module")
def mr(scene, built_lib, grids):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    r = _renderer(scene, grids["occupancy"])
    yield r
    r.close()


@contextlib.contextmanager
def _policy(r, policy):
    try:
        r.set_mlp_accumulator(POLICIES[policy])
        yield
    finally:
        r.set_mlp_accumulator(abi.NSB_MLP_ACC_F16)


def _coords(pw):
    c = np.zeros((pw.shape[0], 7), np.float32)
    c[:, :3] = pw
    c[:, 4:] = 0.5
    return c


def _raw(r, pw):
    """nsb_density at warped positions: the raw fp16 density bits."""
    return np.ascontiguousarray(r.density(_coords(pw))[0]).view(np.uint16)


# ---- density on a grid ----------------------------------------------------------------------------------------------------------
@needs_ref
@pytest.mark.parametrize("name", list(md.QUERIES))
def test_density_on_grid_vs_oracle_and_reference(mr, scene, grids, name):
    res, box, train = md.query(name)
    rows = md.query_rows(res)
    _, pw = mo.grid_positions(res, box, train)
    ref_pos = R("grid_positions", res, box, train, rows)
    np.testing.assert_array_equal(mo.bits(ref_pos[:, :3]), mo.bits(pw[rows]))
    runs = []
    try:
        for gname, grid in grids.items():
            mr.upload_density_grid(grid)
            for policy in POLICIES:
                with _policy(mr, policy):
                    got = mr.density_on_grid(res, box, train).cpu().numpy().reshape(-1)
                    raw = _raw(mr, pw)
                runs.append((f"{gname} {policy}", got, mo.half_to_float(pw, raw, train, grid), R("half_to_float", ref_pos, raw[rows], train, grid)))
    finally:
        mr.upload_density_grid(grids["occupancy"])
    for what, got, exp, ref in runs:
        bad = np.nonzero(mo.bits(got) != mo.bits(exp))[0]
        assert bad.size == 0, f"{what}: {bad.size} points differ from the oracle, first {bad[:8]}: {got[bad[:8]]} vs {exp[bad[:8]]}"
        np.testing.assert_array_equal(mo.bits(got[rows]), mo.bits(ref), err_msg=what)
    assert any((got == mo.FILTERED).any() for _, got, _, _ in runs)


def test_density_on_grid_256x256x512(mr, grids):
    import torch

    res = np.array([256, 256, 512], np.int32)
    box, train = md.query("non_pow2_fox_48")[1:]
    rows = md.query_rows(res, seed=11, k=8192 + 16384)
    got = mr.density_on_grid(res, box, train).reshape(-1)[torch.as_tensor(rows, device="cuda")].cpu().numpy()
    _, pw = mo.grid_positions(res, box, train, rows)
    exp = mo.half_to_float(pw, _raw(mr, pw), train, grids["occupancy"])
    np.testing.assert_array_equal(mo.bits(got), mo.bits(exp))
    assert 0 < (exp == mo.FILTERED).sum() < exp.size


# ---- marching cubes and shading -------------------------------------------------------------------------------------------------
def _mc(r, name, shade=True):
    import torch

    d, box, t = md.FIELDS[name]
    dd = torch.as_tensor(d).cuda()
    nv, ni = r.marching_cubes(dd, md.res_of(name), box, t)
    if shade:
        r.mesh_shade(md.FOX, abi.NSB_ACT_NONE)
    torch.cuda.synchronize()
    return nv, r.mesh_download(nv, ni, shaded=shade)


@needs_ref
@pytest.mark.parametrize("name", list(md.FIELDS))
def test_marching_cubes_and_normals_vs_oracle_and_reference(mr, name):
    d, box, t = md.FIELDS[name]
    Vr, Fr = R("marching_cubes", d, md.res_of(name), box, t)
    nv, m = _mc(mr, name)
    V, F = mo.marching_cubes(d, box[0], box[1], t)
    rows = mo.padded_rows(nv)
    assert nv == V.shape[0] and m["V"].shape[0] == rows and m["F"].shape == F.shape
    np.testing.assert_array_equal(mo.bits(m["V"][:nv]), mo.bits(V))
    assert (mo.bits(m["V"][nv:]) == 0).all() and (mo.bits(m["N"][nv:]) == 0).all()
    np.testing.assert_array_equal(m["F"], F)
    N = mo.normals(m["V"], m["F"], nv, rows)
    bad = np.nonzero((mo.bits(m["N"]) != mo.bits(N)).any(1))[0]
    assert bad.size == 0, f"{bad.size} normals differ, first rows {bad[:8]}: {m['N'][bad[:4]]} vs {N[bad[:4]]}"
    assert Vr.shape == m["V"].shape and Fr.shape == m["F"].shape
    np.testing.assert_array_equal(mo.vertex_multiset(Vr), mo.vertex_multiset(m["V"]))
    np.testing.assert_array_equal(mo.cell_cycle_edges(Vr, Fr), mo.cell_cycle_edges(m["V"], m["F"]))


@pytest.fixture(scope="module")
def scene_mesh(mr):
    """The synthetic scene's iso-surface over a box that is not a power of two: the density grid, its resolution and the threshold."""
    res = np.array([48, 16, 16], np.int32)
    d = mr.density_on_grid(res, md.BOX_NP, md.FOX)
    dn = d.cpu().numpy().reshape(-1)
    return d, res, float(np.median(dn[dn > -10000.0]))


@needs_ref
@pytest.mark.parametrize("linear", [False, True], ids=["srgb", "linear"])
@pytest.mark.parametrize("act", ACTIVATIONS, ids=["none", "relu", "logistic", "exponential"])
def test_colours_vs_reference(mr, scene_mesh, act, linear):
    import torch

    d, res, t = scene_mesh
    nv, ni = mr.marching_cubes(d, res, md.BOX_NP, t)
    assert nv > 100
    coords, runs = None, []
    for policy in POLICIES:
        with _policy(mr, policy):
            mr.mesh_shade(md.FOX, act, linear)
            torch.cuda.synchronize()
            m = mr.mesh_download(nv, ni)
            if coords is None:
                coords = R("color_inputs", m["V"], np.array(md.FOX, np.float32))
            rgbd = mr.inference(coords[:, :7])[:4].view(np.float16).astype(np.float32).T
        runs.append((policy, m, R("srgb", rgbd, act, linear)))
    np.testing.assert_array_equal(mo.bits(coords[:, :7]), mo.bits(mo.color_inputs(m["V"], md.FOX)))
    for policy, m, ref_c in runs:
        np.testing.assert_array_equal(mo.bits(m["C"]), mo.bits(ref_c), err_msg=policy)
        np.testing.assert_array_equal(mo.bits(m["N"]), mo.bits(mo.normals(m["V"], m["F"], nv, m["V"].shape[0])), err_msg=policy)


# ---- empty meshes, context reuse, the index guard -------------------------------------------------------------------------------
@needs_ref
@pytest.mark.parametrize("name", md.EMPTY_FIELDS)
def test_empty_mesh_shades_downloads_and_saves_like_the_reference(mr, tmp_path, name):
    nv, m = _mc(mr, name)
    assert nv == 0 and all(m[k].shape == (0, 3) for k in ("V", "N", "C", "F"))
    for ext in (".ply", ".obj"):
        p = str(tmp_path / ("m" + ext))
        mesh.save_mesh(p, m, 0.33, (0.5, 0.5, 0.5))
        ref_b = R("save_mesh", ext, m["V"], m["N"], m["C"], m["F"], 0.33, np.array([0.5, 0.5, 0.5], np.float32))
        assert open(p, "rb").read() == ref_b.tobytes()


def test_reused_context_matches_fresh_contexts(mr, scene, grids, scene_mesh):
    """big -> small -> empty -> small in one context: every download (V, N, C, F, padding rows included) equals a fresh context's."""
    import torch

    d, res, t = scene_mesh
    big = mr.density_on_grid(np.array([128, 128, 128], np.int32), md.FOX, md.FOX)
    steps = [(big, [128, 128, 128], md.FOX, t)] + [(torch.as_tensor(md.FIELDS[n][0]).cuda(), md.res_of(n), md.FIELDS[n][1], md.FIELDS[n][2])
                                                   for n in ("sphere_cut_by_faces", "all_outside", "random_magnitudes")]

    def run(r, step):
        dd, rr, box, th = step
        nv, ni = r.marching_cubes(dd, rr, box, th)
        r.mesh_shade(md.FOX, abi.NSB_ACT_LOGISTIC)
        torch.cuda.synchronize()
        return nv, r.mesh_download(nv, ni)

    sizes = []
    for step in steps:
        nv, m = run(mr, step)
        fresh = _renderer(scene, grids["occupancy"])
        try:
            nvf, mf = run(fresh, step)
        finally:
            fresh.close()
        assert nv == nvf
        for k in ("V", "N", "C", "F"):
            assert m[k].tobytes() == mf[k].tobytes(), k
        sizes.append(nv)
    assert sizes[0] > sizes[1] > sizes[2] == 0 < sizes[3]


def test_index_overflow_guard(mr):
    """A 720^3 checkerboard has 719^3 cells of 4 triangles each: 1.487e9 triangles, whose indices do not fit 32 bits. nsb_marching_cubes
    rejects it after counting, before it reserves the mesh buffers; the context then has no mesh, and the next small mesh succeeds."""
    import ctypes as C

    import torch

    if torch.cuda.mem_get_info()[0] < 6 << 30:
        pytest.skip("needs 6 GB of free device memory")
    n = 720
    d = torch.empty((n, n, n), dtype=torch.float32, device="cuda")
    i = torch.arange(n, device="cuda", dtype=torch.int32)
    for z in range(n):
        d[z] = torch.where(((i[:, None] + i[None, :] + z) & 1) == 0, 1.0, -1.0)
    res = (C.c_int32 * 3)(n, n, n)
    mn, mx = (C.c_float * 3)(0.0, 0.0, 0.0), (C.c_float * 3)(1.0, 1.0, 1.0)
    nv, ni = C.c_uint64(), C.c_uint64()
    s = torch.cuda.current_stream().cuda_stream
    assert mr.lib.nsb_marching_cubes(mr.ctx, d.data_ptr(), res, mn, mx, 0.0, C.byref(nv), C.byref(ni), s) == abi.NSB_ERR_INVALID
    del d
    torch.cuda.empty_cache()
    tmn, tmx = (C.c_float * 3)(*md.FOX[0]), (C.c_float * 3)(*md.FOX[1])
    assert mr.lib.nsb_mesh_shade(mr.ctx, tmn, tmx, abi.NSB_ACT_NONE, 0, s) == abi.NSB_ERR_STATE
    V = np.zeros((128, 3), np.float32)
    assert mr.lib.nsb_mesh_download(mr.ctx, V.ctypes.data, None, None, 0, None, 0) == abi.NSB_ERR_STATE
    nv, m = _mc(mr, "sphere_cut_by_faces")
    d, box, t = md.FIELDS["sphere_cut_by_faces"]
    V, F = mo.marching_cubes(d, box[0], box[1], t)
    assert nv == V.shape[0] > 0
    np.testing.assert_array_equal(mo.bits(m["V"][:nv]), mo.bits(V))
    np.testing.assert_array_equal(m["F"], F)
