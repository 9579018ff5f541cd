"""The cage tool's "Vanish!" (TetMesh::vanish, tet_mesh.cu:251-363, clear_grid :239-248): the host restatement that nsb_cage_vanish is
tested against (tests/vanish_rule.py: zero and clear where nsb_build_tet_grid's touched-cell bitfield is set) equals the reference's own
vanish byte for byte, grid and bitfield, on every mesh of vanish_rule.meshes. Where the reference build is absent its stored results replay
(tests/ref_golden.py)."""
import os

import numpy as np
import pytest

import vanish_rule as vr
from nerfshop_b200 import synthetic as syn
from oracle import ref_vanish_build
from ref_golden import GOLDEN, _call

_HAVE = ref_vanish_build.build() is not None
MESHES = ["lattice4", "pulled", "coarse", "boundary", "flat"]


@pytest.fixture(scope="module")
def meshes():
    return vr.meshes(syn.make_model(seed=1337))


@pytest.mark.skipif(not _HAVE and not os.path.isdir(os.path.join(GOLDEN, "test_vanish_cpu")), reason="no reference build and no stored results")
@pytest.mark.parametrize("name", MESHES)
def test_host_rule_equals_reference_vanish(meshes, name):
    model = syn.make_model(seed=1337)
    ov, dv, tets = meshes[name]
    grid, bits = vr.inputs(seed=MESHES.index(name))
    stored = _call(_HAVE, vr.reference_vanish, ov, dv, tets, model.aabb_min, model.aabb_max, grid, bits)
    g_ref, b_ref = vr.apply_stored(grid, stored)
    g, b = vr.host_vanish(grid, bits, dv, tets)
    touched = vr.touched_cells(dv, tets)
    per_level = touched.reshape(5, -1).sum(1)
    print(f"\n{name}: {tets.shape[0]} tets, cells touched per cascade {per_level.tolist()}")
    assert touched.any()
    assert np.array_equal(g.view(np.uint32), g_ref.view(np.uint32)), f"{np.count_nonzero(g.view(np.uint32) != g_ref.view(np.uint32))} grid cells differ"
    assert np.array_equal(b, b_ref), f"{np.count_nonzero(b != b_ref)} bitfield bytes differ"


def test_host_rule_without_a_grid_clears_the_same_bits(meshes):
    """A context with a bitfield but no running grid: only the bits change, and they change as with a grid."""
    ov, dv, tets = meshes["pulled"]
    grid, bits = vr.inputs()
    g0, b0 = vr.host_vanish(None, bits, dv, tets)
    g1, b1 = vr.host_vanish(grid, bits, dv, tets)
    assert g0 is None and np.array_equal(b0, b1)


def test_coarse_mesh_reaches_the_coarse_cascades(meshes):
    """The mesh list covers clamped boxes and the coarse cascades: tets that reach cascades 3 and 4 from outside cascades 0 and 1, and a
    zero-volume tet that still touches cells."""
    ov, dv, tets = meshes["coarse"]
    per_level = vr.touched_cells(dv, tets).reshape(5, -1).sum(1)
    assert per_level[3] > 1000 and per_level[4] > 100, per_level.tolist()
    flat = vr.touched_cells(*meshes["flat"][1:]).reshape(5, -1).sum(1)
    assert flat[0] > 0  # a zero-volume tet still touches the cells its faces cross
