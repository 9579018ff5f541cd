"""Mesh extraction on the H100 (nsb_density_on_grid, nsb_marching_cubes, nsb_mesh_shade, nsb_mesh_download) on the synthetic fox-config
scene over its render AABB [-1.5, 2.5]^3. The running density grid is the occupancy bitfield as 0/1 floats, so the filter is active
(-10000) on empty cascade cells. Threshold: the median raw density of the unfiltered points, at which the surface is closed (every
grid point on the box boundary is filtered)."""
import contextlib
import ctypes as C

import numpy as np
import pytest

import mesh_oracle as mo

pytestmark = pytest.mark.gpu

AABB = ((-1.5, -1.5, -1.5), (2.5, 2.5, 2.5))


@pytest.fixture(scope="module")
def mr(scene, built_lib):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nerfshop_b200.renderer import NerfRenderer

    model, occ = scene
    r = NerfRenderer(0)
    r.upload_model(model.desc, model.params)
    r.upload_density_grid(np.unpackbits(occ, bitorder="little").astype(np.float32))
    yield r
    r.close()


def _positions(res):
    """The grid positions and warped coordinates of k_density_on_grid (mesh_oracle.grid_positions: fma(x * (1/res), max - min, min))."""
    return mo.grid_positions((res, res, res), AABB, AABB)


def _density(mr, res):
    return mr.density_on_grid((res, res, res), AABB, AABB).cpu().numpy().reshape(-1)


def _mesh(mr, res, thresh, shade=True):
    import torch

    d = mr.density_on_grid((res, res, res), AABB, AABB)
    nv, ni = mr.marching_cubes(d, (res, res, res), AABB, thresh)
    if shade:
        mr.mesh_shade(AABB, 0)  # rgb activation None: colours are the raw fp16 outputs
    torch.cuda.synchronize()
    return d.cpu().numpy(), mr.mesh_download(nv, ni, shaded=shade), nv


@contextlib.contextmanager
def _policy(mr, policy):
    """The accumulator policy ("f16" or "f32", nsb_set_mlp_accumulator) for a block: nsb_density_on_grid and nsb_mesh_shade follow it like
    nsb_density and nsb_inference. The fp16 default is restored after it."""
    from nerfshop_b200 import abi

    try:
        mr.set_mlp_accumulator(abi.NSB_MLP_ACC_F16 if policy == "f16" else abi.NSB_MLP_ACC_F32)
        yield
    finally:
        mr.set_mlp_accumulator(abi.NSB_MLP_ACC_F16)


def test_density_on_grid_equals_nsb_density_and_filters_empty_cells(mr, scene):
    _density_on_grid_equals_nsb_density(mr, scene, "f16")


def test_density_on_grid_equals_nsb_density_with_fp32_accumulators(mr, scene):
    _density_on_grid_equals_nsb_density(mr, scene, "f32")


def _density_on_grid_equals_nsb_density(mr, scene, policy):
    res = 64
    _, pw = _positions(res)
    coords = np.zeros((pw.shape[0], 7), np.float32)
    coords[:, :3] = pw
    coords[:, 4:] = 0.5
    with _policy(mr, policy):
        got = _density(mr, res)
        raw = mr.density(coords)[0].view(np.float16).astype(np.float32)
    # cascaded_grid_at(unwarp(warp(p)), density_grid, mip_from_pos) of the occupancy as 0/1
    model, occ = scene
    empty = mo.filtered(pw, AABB, np.unpackbits(occ, bitorder="little").astype(np.float32))
    assert 0 < empty.sum() < empty.size
    np.testing.assert_array_equal(got[~empty].view(np.uint32), raw[~empty].view(np.uint32))
    assert (got[empty] == -10000.0).all()


def _thresh(d):
    v = d[d > -10000.0]
    return float(np.median(v))


def test_marching_cubes_matches_the_oracle_and_is_deterministic(mr):
    res = 128
    d0, m0, nv = _mesh(mr, res, 0.0, shade=False)
    t = _thresh(d0)
    d, m, nv = _mesh(mr, res, t)
    V, F = mo.marching_cubes(d.reshape(res, res, res), AABB[0], AABB[1], t)
    assert nv == V.shape[0] > 1000 and m["V"].shape[0] == ((nv + 127) // 128) * 128
    np.testing.assert_array_equal(m["V"][:nv].view(np.uint32), V.view(np.uint32))
    assert (m["V"][nv:] == 0).all() and (m["N"][nv:] == 0).all()
    np.testing.assert_array_equal(m["F"], F)
    assert mo.edge_manifold(F)
    _, m2, _ = _mesh(mr, res, t)
    for k in ("V", "N", "C", "F"):
        assert m[k].tobytes() == m2[k].tobytes(), k


def test_normals_and_colours(mr):
    _normals_and_colours(mr, "f16")


def test_normals_and_colours_with_fp32_accumulators(mr):
    _normals_and_colours(mr, "f32")


def _normals_and_colours(mr, policy):
    res = 64
    with _policy(mr, policy):
        d0 = _density(mr, res)
        t = _thresh(d0)
        d, m, nv = _mesh(mr, res, t)
    V, N, Cc, F = m["V"], m["N"], m["C"], m["F"].astype(np.int64)
    # normals: (pb - pa) x (pa - pc) per triangle in its FMA form, summed in ascending triangle order, bit for bit; zero padding rows
    np.testing.assert_array_equal(mo.bits(N), mo.bits(mo.normals(V, F, nv, V.shape[0])))
    # colours: the network at {warp(pos), warp(normalize(pos - 0.5))} (mesh_oracle.color_inputs), every row, bit for bit
    with _policy(mr, policy):
        raw = mr.inference(mo.color_inputs(V, AABB))[:3].view(np.float16).astype(np.float32).T
    np.testing.assert_array_equal(Cc.view(np.uint32), raw.view(np.uint32))


def test_256_mesh_is_edge_manifold_and_reused_context_matches_fresh(mr, scene):
    from nerfshop_b200.renderer import NerfRenderer

    d64 = _density(mr, 64)
    t = _thresh(d64)
    _mesh(mr, 64, t)
    d, m, nv = _mesh(mr, 256, t)
    dd = d.reshape(256, 256, 256)
    assert (dd[[0, -1]] <= t).all() and (dd[:, [0, -1]] <= t).all() and (dd[:, :, [0, -1]] <= t).all()
    assert nv > 0 and mo.edge_manifold(m["F"])
    model, occ = scene
    fresh = NerfRenderer(0)
    fresh.upload_model(model.desc, model.params)
    fresh.upload_density_grid(np.unpackbits(occ, bitorder="little").astype(np.float32))
    _, mf, nvf = _mesh(fresh, 256, t)
    fresh.close()
    assert nvf == nv
    for k in ("V", "N", "C", "F"):
        assert m[k].tobytes() == mf[k].tobytes(), k


def test_status_codes(scene, built_lib):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nerfshop_b200 import abi
    from nerfshop_b200.renderer import NerfRenderer

    model, occ = scene
    r = NerfRenderer(0)
    out = torch.zeros(16 ** 3, device="cuda")
    q = abi.NsbGridQuery()
    q.res[:] = [16, 16, 16]
    q.aabb_min[:] = q.train_aabb_min[:] = AABB[0]
    q.aabb_max[:] = q.train_aabb_max[:] = AABB[1]
    assert r.lib.nsb_density_on_grid(r.ctx, C.byref(q), out.data_ptr(), None) == abi.NSB_ERR_STATE  # no model
    r.upload_model(model.desc, model.params)
    assert r.lib.nsb_density_on_grid(r.ctx, C.byref(q), out.data_ptr(), None) == abi.NSB_ERR_STATE  # no density grid
    r.upload_density_grid(np.unpackbits(occ, bitorder="little").astype(np.float32))
    assert r.lib.nsb_density_on_grid(r.ctx, C.byref(q), out.data_ptr(), None) == abi.NSB_OK
    for bad in ([17, 16, 16], [16, 0, 16], [16, 16, -16]):
        q.res[:] = bad
        assert r.lib.nsb_density_on_grid(r.ctx, C.byref(q), out.data_ptr(), None) == abi.NSB_ERR_INVALID
        res = (C.c_int32 * 3)(*bad)
        mn, mx = (C.c_float * 3)(*AABB[0]), (C.c_float * 3)(*AABB[1])
        assert r.lib.nsb_marching_cubes(r.ctx, out.data_ptr(), res, mn, mx, 0.0, None, None, None) == abi.NSB_ERR_INVALID
    assert r.lib.nsb_mesh_download(r.ctx, None, None, None, 0, None, 0) == abi.NSB_ERR_STATE  # no mesh yet
    d = r.density_on_grid((64, 64, 64), AABB, AABB)
    nv, ni = r.marching_cubes(d, (64, 64, 64), AABB, _thresh(d.cpu().numpy().reshape(-1)))
    assert nv > 0 and ni > 0
    V = np.zeros((nv + 128, 3), np.float32)
    F = np.zeros(ni, np.uint32)
    assert r.lib.nsb_mesh_download(r.ctx, None, V.ctypes.data, None, nv, None, 0) == abi.NSB_ERR_STATE  # normals before nsb_mesh_shade
    assert r.lib.nsb_mesh_download(r.ctx, V.ctypes.data, None, None, ((nv + 127) // 128) * 128 + 1, None, 0) == abi.NSB_ERR_INVALID
    assert r.lib.nsb_mesh_download(r.ctx, None, None, None, 0, F.ctypes.data, ni - 1) == abi.NSB_ERR_INVALID
    assert r.lib.nsb_mesh_download(r.ctx, V.ctypes.data, None, None, nv, F.ctypes.data, ni) == abi.NSB_OK
    r.close()
