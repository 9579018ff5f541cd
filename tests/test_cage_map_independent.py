"""CPU: an independent numpy restatement of EditOperator::map_rays for a cage (interpolate_tet, cage_deformation.cu:197-269;
point_in_tet / bary_tet, selection_utils.h:10-47) that does NOT use the lookup table: every tet is tested, the lowest-index containing
tet wins (= the first entry of the sample's cell list, whose entries are in ascending tet order). The rule lives in tests/edit_domain.py
(map_rays_lut_free). Against the oracle's LUT-driven map_rays: positions, directions and the empty mask bit for bit. Also pins the LUT's
completeness on these samples."""
import numpy as np

import edit_domain as ed
import edit_fixtures as fx
from conftest import random_coords
from oracle import oracle as orc

F32 = np.float32


def test_numpy_cage_map_equals_the_oracle(scene):
    model, occ = scene
    op = fx.e1(model)[0]
    o = orc.Oracle(model.desc, model.params, occ, [op.to_op()])
    rng = np.random.default_rng(4)
    n = 700
    c = random_coords(n, 9)
    centre, half = np.array([0.55, 0.62, 0.78], F32), np.array([0.3, 0.26, 0.26], F32)
    p = centre + (rng.random((n, 3)).astype(F32) * 2 - 1) * half
    c[:, :3] = (p - model.aabb_min) / (model.aabb_max - model.aabb_min)
    ref, mref = o.map_rays(c)
    got, mgot = ed.map_rays_lut_free([op], c)
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32)), np.nonzero((got != ref).any(1))[0][:10]
    assert np.array_equal(mgot, mref)
    moved = (got[:, :3] != c[:, :3]).any(1)
    assert moved.sum() > 100 and mgot.sum() >= 1
