"""Mesh extraction against the reference's own code (oracle/_ref/libnerfshop_ref_mesh_cuda.so: marching_cubes.cu and the grid / colour
kernels of testbed_nerf.cu compiled by nvcc), through tests/ref_golden.py: where that build is absent the stored results replay.

Scene: the synthetic fox-config model, train AABB [-1.5, 2.5]^3, the occupancy as the running density grid (0/1 floats). The box meshed
has extents that are not powers of two and a 48-point axis, so x * (1/res), the AABB scale and the vertex scale are rounded products
and the FMA contraction matters. This repository's nsb_density / nsb_inference stand in for tiny-cuda-nn between the reference's kernels.
"""
import numpy as np
import pytest

import mesh_oracle as mo
import ref_golden as rg
from nerfshop_b200 import abi, mesh
from oracle import ref_mesh, ref_mesh_build

HAVE = ref_mesh_build.build() is not None
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not (HAVE or rg._stored("test_gpu_mesh_ref")),
                                                  reason="neither oracle/_ref nor stored reference results (tests/golden/ref/)")]

TRAIN = np.array([[-1.5, -1.5, -1.5], [2.5, 2.5, 2.5]], np.float32)
BOX = np.array([[-1.3, -1.1, -0.9], [2.2, 2.1, 2.4]], np.float32)
RES = np.array([48, 16, 16], np.int32)


@pytest.fixture(autouse=True)
def _device_for_the_live_reference():
    """The reference build runs on the GPU; its stored results replay anywhere."""
    import torch

    if HAVE and not torch.cuda.is_available():
        pytest.skip("no CUDA device for the reference build")


def R(name, *args):
    """The reference's result (or its stored replay)."""
    return rg._call(HAVE, getattr(ref_mesh, name) if HAVE else None, *args)


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


def _ours_mesh(mr, rgb_activation=abi.NSB_ACT_LOGISTIC, linear_colors=False):
    import torch

    d = mr.density_on_grid(RES, BOX, TRAIN)
    dn = d.cpu().numpy().reshape(-1)
    t = float(np.median(dn[dn > -10000.0]))
    nv, ni = mr.marching_cubes(d, RES, BOX, t)
    mr.mesh_shade(TRAIN, rgb_activation, linear_colors)
    torch.cuda.synchronize()
    return dn, t, nv, mr.mesh_download(nv, ni)


def test_density_on_grid_vs_reference_with_filter_on_and_off(mr, scene):
    model, occ = scene
    pos = R("grid_positions", RES, BOX, TRAIN)
    coords = np.zeros((pos.shape[0], 7), np.float32)
    coords[:, :3] = pos[:, :3]
    coords[:, 4:] = 0.5
    raw = mr.density(coords)[0]  # nsb_density standing in for NerfNetwork::density
    grid = np.unpackbits(occ, bitorder="little").astype(np.float32)
    ref_on = R("half_to_float", pos, raw, TRAIN, grid)
    ref_off = R("half_to_float", pos, raw, TRAIN)
    ours = mr.density_on_grid(RES, BOX, TRAIN).cpu().numpy().reshape(-1)
    filtered = ref_on == -10000.0
    assert 0 < filtered.sum() < filtered.size  # both sides of the filter are checked
    np.testing.assert_array_equal(ours.view(np.uint32), ref_on.view(np.uint32))
    np.testing.assert_array_equal(ours[~filtered].view(np.uint32), ref_off[~filtered].view(np.uint32))


def test_single_cell_cycles_vs_reference_gen_faces():
    """All 256 configurations of one cell through marching_cubes_gpu: the boundary cycles of its triangles, with their direction, equal
    the generated table's (the list of configurations allowed to differ is empty)."""
    mids = {}
    for e, (a, b) in enumerate(mo.gen_mc_table.EDGES):
        p = (np.array(mo.CORNER[a], np.float32) + np.array(mo.CORNER[b], np.float32)) * np.float32(0.5)
        mids[tuple(p.tolist())] = e
    differ = []
    for cfg in range(1, 255):
        d = np.zeros((2, 2, 2), np.float32)
        for k, (x, y, z) in enumerate(mo.CORNER):
            d[z, y, x] = 1.0 if (cfg >> k) & 1 else -1.0
        V, F = R("marching_cubes", d, np.array([2, 2, 2], np.int32), np.array([[0, 0, 0], [2, 2, 2]], np.float32), 0.0)
        edge = [mids.get(tuple(v.tolist()), -1) for v in V]
        tris = [tuple(edge[i] for i in t) for t in F]
        if mo.boundary_cycles(tris) != mo.boundary_cycles(mo.TABLE[cfg]):
            differ.append(cfg)
    assert differ == []


def test_vertex_multiset_and_triangle_count_vs_reference_marching_cubes(mr):
    import torch

    d = mr.density_on_grid(RES, BOX, TRAIN)
    dn = d.cpu().numpy().reshape(-1)
    t = float(np.median(dn[dn > -10000.0]))
    nv, ni = mr.marching_cubes(d, RES, BOX, t)
    torch.cuda.synchronize()
    ours = mr.mesh_download(nv, ni, shaded=False)
    V, F = R("marching_cubes", dn, RES, BOX, t)
    assert nv > 100 and V.shape[0] == ours["V"].shape[0] and F.shape[0] == ni // 3  # same padded rows, same number of triangles
    key = lambda a: np.sort(np.ascontiguousarray(a).view(np.uint32).view([("x", "<u4"), ("y", "<u4"), ("z", "<u4")]).reshape(-1))
    assert (key(ours["V"]) == key(V)).all()  # the same edge crossings, bit for bit (padding rows at the origin included)


def test_normals_colours_and_padding_vs_reference(mr):
    """Colours bit for bit through generate_nerf_network_inputs_from_positions + the network + extract_srgb_with_activation, for every row
    including the padding; normals against compute_mesh_1ring on the same mesh (its float atomics sum in arbitrary order, so the
    comparison is in angle), and zero on the padding rows."""
    for act, lin in ((abi.NSB_ACT_LOGISTIC, False), (abi.NSB_ACT_LOGISTIC, True), (abi.NSB_ACT_NONE, False)):
        _, _, nv, m = _ours_mesh(mr, act, lin)
        coords = R("color_inputs", m["V"], TRAIN)
        rgbd = mr.inference(coords[:, :7])[:4].view(np.float16).astype(np.float32).T
        ref_c = R("srgb", rgbd, act, lin)
        np.testing.assert_array_equal(m["C"].view(np.uint32), ref_c.view(np.uint32))
    ref_n = R("normals", m["V"], m["F"])
    a, b = m["N"][:nv].astype(np.float64), ref_n[:nv].astype(np.float64)
    na, nb = np.linalg.norm(a, axis=1), np.linalg.norm(b, axis=1)
    zero = (na == 0) | (nb == 0)  # every triangle at the vertex degenerate (crossings at a grid point): the sum is 0 or cancels to rounding
    assert zero.mean() < 0.01 and (na[zero] < 1e-9).all() and (nb[zero] < 1e-9).all()
    cos = np.einsum("ij,ij->i", a[~zero], b[~zero]) / (na[~zero] * nb[~zero])
    assert (cos > 1 - 1e-6).all()
    assert (m["N"][nv:] == 0).all() and (ref_n[nv:] == 0).all()


@pytest.mark.parametrize("ext", [".ply", ".obj"])
def test_save_mesh_bytes_vs_reference(mr, tmp_path, ext):
    _, _, nv, m = _ours_mesh(mr)
    p = str(tmp_path / ("m" + ext))
    mesh.save_mesh(p, m, 0.33, (0.5, 0.5, 0.5))
    ours = np.frombuffer(open(p, "rb").read(), np.uint8)
    ref_b = R("save_mesh", ext, m["V"], m["N"], m["C"], m["F"], 0.33, np.array([0.5, 0.5, 0.5], np.float32))
    assert ours.tobytes() == ref_b.tobytes()


def test_get_marching_cubes_res_vs_reference():
    for res_1d, box in ((256, TRAIN), (100, BOX), (512, np.array([[0, 0, 0], [1.0, 0.5, 0.3]], np.float32)), (37, np.array([[-0.2, 0.1, 0.3], [0.9, 0.4, 1.7]], np.float32))):
        np.testing.assert_array_equal(mesh.get_marching_cubes_res(res_1d, box), R("get_marching_cubes_res", res_1d, box))
