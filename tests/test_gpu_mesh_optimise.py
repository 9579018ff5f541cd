"""nsb_mesh_optimise (Testbed::optimise_mesh_step) on the H100, on the synthetic scene of test_gpu_mesh.py (render AABB [-1.5, 2.5]^3, the
running density grid = the occupancy bitfield as 0/1, threshold = the median raw density of the unfiltered grid points). One step is the
CPU mirror's bit for bit when the mirror is fed the device's density and gradient at the same positions; 20 steps are deterministic; the
density term pulls the vertices towards the iso-surface."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

AABB = ((-1.5, -1.5, -1.5), (2.5, 2.5, 2.5))
RES = 64


def _renderer(scene):
    from nerfshop_b200.renderer import NerfRenderer

    model, occ = scene
    r = NerfRenderer(0)
    r.upload_model(model.desc, model.params)
    r.upload_density_grid(np.unpackbits(occ, bitorder="little").astype(np.float32))
    return r


@pytest.fixture(scope="module")
def mr(scene, built_lib):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    r = _renderer(scene)
    yield r
    r.close()


def _thresh(r):
    d = r.density_on_grid((RES, RES, RES), AABB, AABB).cpu().numpy().reshape(-1)
    return float(np.median(d[d > -10000.0]))


def _remesh(r, t):
    d = r.density_on_grid((RES, RES, RES), AABB, AABB)
    return r.marching_cubes(d, (RES, RES, RES), AABB, t)


def _download(r, nv, ni, normals=True):
    """Vertex rows (padding included), normals and faces, without colours (the mesh need not be shaded)."""
    rows = (nv + 127) // 128 * 128
    V, N, F = np.zeros((rows, 3), np.float32), np.zeros((rows, 3), np.float32), np.zeros((ni // 3, 3), np.uint32)
    st = r.lib.nsb_mesh_download(r.ctx, V.ctypes.data, N.ctypes.data if normals else None, None, rows, F.ctypes.data, F.size)
    assert st == 0, r.lib.nsb_last_error()
    return V, N, F


def _coords(V):
    c = np.zeros((V.shape[0], 7), np.float32)
    c[:, :3] = (V - np.float32(-1.5)) / np.float32(4.0)  # warp_position; exact for this power-of-two box
    c[:, 4:] = 0.5
    return c


def test_one_step_equals_the_mirror(mr):
    from oracle import mesh_opt_oracle as mo

    t = _thresh(mr)
    nv, ni = _remesh(mr, t)
    V0, _, F0 = _download(mr, nv, ni, normals=False)
    assert nv > 1000 and V0.shape[0] > nv
    grad, dens = mr.density_gradient(_coords(V0))
    mr.mesh_optimise(1, t, AABB)
    V1, N1, F1 = _download(mr, nv, ni)
    np.testing.assert_array_equal(F1, F0)
    P, N, (m1, m2, steps) = mo.mesh_opt_step(V0, F0, dens, grad, t, 2048.0, 128.0, 1.0)
    np.testing.assert_array_equal(N1.view(np.uint32), N.view(np.uint32))
    np.testing.assert_array_equal(V1.view(np.uint32), P.view(np.uint32))
    assert (V1[nv:] != 0).any()  # the padding rows are optimised too, and move
    assert (np.abs(V1 - V0) <= 1.01e-4).all() and (V1 != V0).mean() > 0.9


def test_twenty_steps_are_deterministic_and_keep_the_indices(mr, scene):
    t = _thresh(mr)
    out = []
    for r in (mr, _renderer(scene)):
        nv, ni = _remesh(r, t)
        _, _, F0 = _download(r, nv, ni, normals=False)
        r.mesh_optimise(20, t, AABB)
        V, N, F = _download(r, nv, ni)
        np.testing.assert_array_equal(F, F0)
        out.append((V, N))
        if r is not mr:
            r.close()
    assert out[0][0].tobytes() == out[1][0].tobytes() and out[0][1].tobytes() == out[1][1].tobytes()


def test_density_term_moves_vertices_towards_the_iso_surface(mr):
    t = _thresh(mr)
    nv, ni = _remesh(mr, t)
    V0, _, _ = _download(mr, nv, ni, normals=False)
    mr.mesh_optimise(20, t, AABB, smooth_amount=0.0, density_amount=128.0, inflate_amount=0.0)
    V1, _, _ = _download(mr, nv, ni, normals=False)
    e0 = np.abs(mr.density(_coords(V0[:nv]))[0].view(np.float16).astype(np.float64) - t).mean()
    e1 = np.abs(mr.density(_coords(V1[:nv]))[0].view(np.float16).astype(np.float64) - t).mean()
    print(f"\nmean |raw density - thresh| at {nv} vertices: {e0:.5f} -> {e1:.5f} after 20 steps")
    assert e1 < e0


def test_remesh_then_optimise_equals_a_fresh_context(mr, scene):
    t = _thresh(mr)
    _remesh(mr, t)
    mr.mesh_optimise(5, t, AABB)
    nv, ni = _remesh(mr, t)
    mr.mesh_optimise(5, t, AABB)
    V, N, F = _download(mr, nv, ni)
    fresh = _renderer(scene)
    nvf, nif = _remesh(fresh, t)
    fresh.mesh_optimise(5, t, AABB)
    Vf, Nf, Ff = _download(fresh, nvf, nif)
    fresh.close()
    assert (nv, ni) == (nvf, nif)
    assert V.tobytes() == Vf.tobytes() and N.tobytes() == Nf.tobytes() and F.tobytes() == Ff.tobytes()


def test_status_codes(scene, built_lib):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nerfshop_b200 import abi
    from nerfshop_b200.renderer import NerfRenderer

    model, occ = scene
    p = abi.NsbMeshOptimise()
    p.thresh, p.smooth_amount, p.density_amount, p.inflate_amount = 0.0, 2048.0, 128.0, 1.0
    p.train_aabb_min[:], p.train_aabb_max[:] = AABB
    r = NerfRenderer(0)
    assert r.lib.nsb_mesh_optimise(r.ctx, C.byref(p), 1, None) == abi.NSB_ERR_STATE  # no model
    r.upload_model(model.desc, model.params)
    assert r.lib.nsb_mesh_optimise(r.ctx, C.byref(p), 1, None) == abi.NSB_ERR_STATE  # no mesh
    r.upload_density_grid(np.unpackbits(occ, bitorder="little").astype(np.float32))
    nv, ni = _remesh(r, _thresh(r))
    assert r.lib.nsb_mesh_optimise(r.ctx, None, 1, None) == abi.NSB_ERR_INVALID
    V = np.zeros((nv, 3), np.float32)
    assert r.lib.nsb_mesh_download(r.ctx, None, V.ctypes.data, None, nv, None, 0) == abi.NSB_ERR_STATE  # no normals yet
    assert r.lib.nsb_mesh_optimise(r.ctx, C.byref(p), 1, None) == abi.NSB_OK
    assert r.lib.nsb_mesh_download(r.ctx, None, V.ctypes.data, None, nv, None, 0) == abi.NSB_OK  # the optimiser leaves normals
    assert r.lib.nsb_mesh_download(r.ctx, None, None, V.ctypes.data, nv, None, 0) == abi.NSB_ERR_STATE  # but no colours
    r.close()
