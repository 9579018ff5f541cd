"""Marching-cubes table, mesh topology on analytic fields, get_marching_cubes_res and save_mesh — no GPU needed."""
import os

import numpy as np

import mesh_oracle as mo
from nerfshop_b200 import mesh


def test_generator_reproduces_committed_header():
    with open(mo.gen_mc_table.OUT) as fh:
        assert fh.read() == mo.gen_mc_table.render()


def test_table_rows_triangulate_exactly_the_face_cycles():
    """For all 256 configurations the triangles' boundary is the set of cycles chained from the face segments, with its direction."""
    for cfg in range(256):
        cyc = frozenset(tuple(c[c.index(min(c)):] + c[:c.index(min(c))]) for c in mo.gen_mc_table.cycles(cfg))
        assert mo.boundary_cycles(mo.TABLE[cfg]) == cyc, cfg
    assert mo.TABLE[1] == [(0, 8, 3)]  # the reference's winding: corner 0 inside, normal (by the right-hand rule) pointing away from it
    assert max(len(t) for t in mo.TABLE) == 5


def test_complementary_configurations_are_reversed_where_no_face_is_decided():
    """Swapping inside and outside reverses every cycle when no face has four crossings (the face rule is not symmetric there)."""
    four = set(mo.gen_mc_table.four_crossing_configs())
    for cfg in range(1, 255):
        if cfg in four:
            continue
        rev = frozenset(tuple(c[::-1][-1:] + c[::-1][:-1]) for c in mo.boundary_cycles(mo.TABLE[cfg]))
        rev = frozenset(tuple(c[c.index(min(c)):] + c[:c.index(min(c))]) for c in rev)
        assert mo.boundary_cycles(mo.TABLE[255 - cfg]) == rev, cfg


def _grid(n, f):
    t = (np.arange(n, dtype=np.float32) + 0.5) / n * 2 - 1
    z, y, x = np.meshgrid(t, t, t, indexing="ij")
    return f(x, y, z).astype(np.float32)


def test_sphere_is_closed_with_euler_characteristic_2():
    d = _grid(48, lambda x, y, z: 0.7 - np.sqrt(x * x + y * y + z * z))
    V, F = mo.marching_cubes(d, (-1, -1, -1), (1, 1, 1), 0.0)
    assert F.shape[0] > 1000 and mo.edge_manifold(F) and mo.euler_characteristic(F) == 2
    c = V[F].mean(1)
    n = np.cross(V[F[:, 1]] - V[F[:, 0]], V[F[:, 0]] - V[F[:, 2]])  # accumulate_1ring's (pb - pa) x (pa - pc)
    assert (np.einsum("ij,ij->i", n, c) > 0).mean() > 0.99  # the reference's orientation: normals point out of the inside


def test_torus_is_closed_with_euler_characteristic_0():
    d = _grid(64, lambda x, y, z: 0.25 - np.sqrt((np.sqrt(x * x + y * y) - 0.55) ** 2 + z * z))
    _, F = mo.marching_cubes(d, (-1, -1, -1), (1, 1, 1), 0.0)
    assert F.shape[0] > 1000 and mo.edge_manifold(F) and mo.euler_characteristic(F) == 0


def test_seeded_noise_is_edge_manifold():
    rng = np.random.default_rng(7)
    d = rng.standard_normal((40, 40, 40)).astype(np.float32)
    d[0, :, :] = d[-1, :, :] = d[:, 0, :] = d[:, -1, :] = d[:, :, 0] = d[:, :, -1] = -1.0  # kept clear of the boundary
    _, F = mo.marching_cubes(d, (0, 0, 0), (1, 1, 1), 0.0)
    assert F.shape[0] > 10000 and mo.edge_manifold(F)


def test_get_marching_cubes_res():
    np.testing.assert_array_equal(mesh.get_marching_cubes_res(256, ((-1.5, -1.5, -1.5), (2.5, 2.5, 2.5))), [256, 256, 256])
    np.testing.assert_array_equal(mesh.get_marching_cubes_res(100, ((0, 0, 0), (1.0, 0.5, 0.3))), [112, 64, 32])


def _small_mesh():
    V = np.zeros((128, 3), np.float32)
    V[:3] = [[0.5, 0.25, 0.125], [1.0, 0.5, 0.0], [0.0, 1.0, 0.75]]
    N = np.zeros((128, 3), np.float32)
    N[:3] = [[0, 0, 2], [3, 4, 0], [-1, 0, 0]]
    C = np.full((128, 3), 0.5, np.float32)
    C[0] = [1.5, -0.25, 0.999]
    return dict(V=V, N=N, C=C, F=np.array([[0, 1, 2]], np.int32))


def test_save_mesh_ply_format(tmp_path):
    p = str(tmp_path / "m.ply")
    mesh.save_mesh(p, _small_mesh(), 0.33, (0.5, 0.5, 0.5))
    lines = open(p).read().split("\n")
    assert lines[0] == "ply" and lines[3] == "element vertex 128" and lines[13] == "element face 1" and lines[15] == "end_header"
    assert lines[16] == "0.00000 -0.75758 -1.13636 0.000 0.000 1.000 255 0 254"
    assert lines[17] == "1.51515 0.00000 -1.51515 0.600 0.800 0.000 127 127 127"
    assert lines[16 + 127] == "-1.51515 -1.51515 -1.51515 0.000 0.000 0.000 127 127 127"  # a padding row
    assert lines[16 + 128] == "3 2 1 0"


def test_save_mesh_obj_format(tmp_path):
    p = str(tmp_path / "m.obj")
    mesh.save_mesh(p, _small_mesh(), 0.33, (0.5, 0.5, 0.5))
    lines = open(p).read().split("\n")
    assert lines[0] == "v 0.00000 -0.75758 -1.13636 1.000 0.000 0.999"
    assert lines[128] == "vn 0.00000 0.00000 1.00000"
    assert lines[256] == "f 3//3 2//2 1//1" and lines[257] == ""
