"""The mesh oracle (tests/mesh_oracle.py) against the reference's own mesh-extraction kernels over the domain of tests/mesh_domain.py.

The reference's kernels (marching_cubes.cu, the grid and colour kernels of testbed_nerf.cu) run through
oracle/_ref/libnerfshop_ref_mesh_cuda.so where it is built and a GPU is present; elsewhere their stored results (tests/golden/ref/)
replay, so this file runs on any machine.

  * marching cubes on every field: the vertex multiset bit for bit (all NaNs equal), the counts, zero padding rows, and the cells'
    boundary cycles with their direction (mesh_oracle.cell_cycle_edges: the reference's table triangulates some cycles differently,
    and it orders vertices and triangles by atomics; tests/test_gpu_mesh_domain.py pins the device's order to the oracle);
  * the grid positions of every query, bit for bit, and the filter of grid_samples_half_to_float on synthetic fp16 densities;
  * the colour inputs of every field's mesh, padding rows at the origin and a vertex at the AABB centre included.
"""
import numpy as np
import pytest

import mesh_domain as md
import mesh_oracle as mo
import ref_golden as rg
from oracle import ref_mesh, ref_mesh_build

HAVE = ref_mesh_build.build() is not None
pytestmark = pytest.mark.skipif(not (HAVE or rg._stored("test_mesh_domain_cpu")),
                                reason="neither oracle/_ref nor stored reference results (tests/golden/ref/)")


def _live():
    if not HAVE:
        return False
    import torch

    return torch.cuda.is_available()


def R(name, *args):
    """The reference's result: live where its build and a GPU are present, else the stored replay. Never a row sample."""
    v = rg._call(_live(), getattr(ref_mesh, name), *args)
    for a in v if isinstance(v, tuple) else (v,):
        assert not isinstance(a, rg.Sampled)
    return v


def test_random_fields_reach_every_configuration():
    assert md.config_coverage() == set(range(1, 255))


def test_checkerboard_has_four_triangles_per_cell():
    d, box, t = md.FIELDS["checkerboard"]
    _, F = mo.marching_cubes(d, box[0], box[1], t)
    assert F.shape[0] == 4 * 15 ** 3


@pytest.mark.parametrize("name", list(md.FIELDS))
def test_marching_cubes_vs_reference(name):
    d, box, t = md.FIELDS[name]
    V, F = mo.marching_cubes(d, box[0], box[1], t)
    Vr, Fr = R("marching_cubes", d, md.res_of(name), box, t)
    nv = V.shape[0]
    assert Vr.shape[0] == mo.padded_rows(nv) and Fr.shape == F.shape
    assert (nv == 0) == (name in md.EMPTY_FIELDS)
    assert (mo.bits(Vr[nv:]) == 0).all()  # the padding rows sit at +0, +0, +0
    assert (Fr < nv).all()
    np.testing.assert_array_equal(mo.vertex_multiset(Vr[:nv]), mo.vertex_multiset(V))
    np.testing.assert_array_equal(mo.cell_cycle_edges(Vr, Fr), mo.cell_cycle_edges(V, F))


@pytest.mark.parametrize("name", list(md.FIELDS))
def test_color_inputs_vs_reference(name):
    """On the field's mesh as the device stores it (vertex rows rounded up to 128, the padding at the origin) plus a vertex at the centre
    (0.5, 0.5, 0.5), whose direction has norm 0 and stays unnormalised; the train AABB is neither cubic nor a power of two."""
    d, box, t = md.FIELDS[name]
    V, _ = mo.marching_cubes(d, box[0], box[1], t)
    rows = np.zeros((mo.padded_rows(V.shape[0]) + 1, 3), np.float32)
    rows[:V.shape[0]] = V
    rows[-1] = 0.5
    ref = R("color_inputs", rows, np.array(md.TRAIN_NP, np.float32))
    np.testing.assert_array_equal(mo.bits(mo.color_inputs(rows, md.TRAIN_NP)), mo.bits(ref[:, :7]))


@pytest.mark.parametrize("name", list(md.QUERIES))
def test_grid_positions_vs_reference(name):
    res, box, train = md.query(name)
    rows = md.query_rows(res)
    ref = R("grid_positions", res, box, train, rows)
    _, pw = mo.grid_positions(res, box, train, rows)
    np.testing.assert_array_equal(mo.bits(pw), mo.bits(ref[:, :3]))


@pytest.mark.parametrize("name", list(md.QUERIES))
def test_filter_vs_reference_half_to_float(scene, name):
    """Synthetic fp16 densities (every finite fp16 value may occur) through grid_samples_half_to_float, without a density grid and with each
    of tests/mesh_domain.py's density grids."""
    res, box, train = md.query(name)
    rows = md.query_rows(res)
    ref_pos = R("grid_positions", res, box, train, rows)
    _, pw = mo.grid_positions(res, box, train, rows)
    raw = np.random.default_rng(rows.size).integers(0, 0x7c00, rows.size, dtype=np.uint16) | (
        np.random.default_rng(rows.size + 1).integers(0, 2, rows.size, dtype=np.uint16) << np.uint16(15))
    np.testing.assert_array_equal(mo.bits(R("half_to_float", ref_pos, raw, train)), mo.bits(mo.half_to_float(pw, raw, train)))
    seen = 0
    for grid in md.density_grids(scene[1]).values():
        ours = mo.half_to_float(pw, raw, train, grid)
        np.testing.assert_array_equal(mo.bits(R("half_to_float", ref_pos, raw, train, grid)), mo.bits(ours))
        seen += (ours == mo.FILTERED).any()
    assert seen  # the filter applies somewhere
