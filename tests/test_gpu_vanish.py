"""The cage tool's "Vanish!" on the device: nsb_cage_vanish against the host restatement of TetMesh::vanish (tests/vanish_rule.py, pinned
to the reference's own vanish by tests/test_vanish_cpu.py). The cell test is integer / pinned-fp32 work, so grid and bitfield must agree
bit for bit; frames and occupancy updates that follow are compared with the oracle as the render and grid-update tests compare them."""
import ctypes as C

import numpy as np
import pytest

import edit_fixtures as fx
import vanish_rule as vr
from nerfshop_b200 import abi, editing
from nerfshop_b200 import synthetic as syn
from nerfshop_b200.rng import Pcg32
from oracle import oracle as orc
from test_gpu_grid_update import _compare as compare_grid_update
from test_gpu_parity import _compare_frames
from test_grid_update_cpu import grid_params

pytestmark = pytest.mark.gpu


@pytest.fixture
def fresh(scene, built_lib):
    """A context of its own per test (one without a running grid must never have had one)."""
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nerfshop_b200.renderer import NerfRenderer

    model, _ = scene
    r = NerfRenderer(0)
    r.upload_model(model.desc, model.params)
    yield r
    r.close()


def as_operator(model, ov, dv, tets):
    """A cage operator whose tets sit exactly at dv (a box cage around them; the MVC weights are not used)."""
    lo, hi = np.asarray(ov).min(0) - 0.05, np.asarray(ov).max(0) + 0.05
    op = editing.CageDeformation(model.aabb_min, model.aabb_max, *editing.box_cage(lo, hi), ov, tets)
    op.vertices = np.array(dv, np.float32)
    op.lut_offsets = np.zeros(abi.NSB_GRID_CELLS + 1, np.uint32)
    op.lut_idx = op._grid(op.vertices, op.lut_offsets, None)
    return op


def changed_cells(g0, b0, g1, b1):
    bits_changed = np.unpackbits(b0 ^ b1, bitorder="little").astype(bool)
    if g0 is None:
        return bits_changed
    return bits_changed | (g0.view(np.uint32) != g1.view(np.uint32))


def _vanish_and_check(r, op_index, verts, tets, g0, b0, with_grid, stream=0):
    n = r.cage_vanish(op_index, count=True, stream=stream)
    g1, b1 = r.download_density_grid(want_grid=with_grid)
    g_host, b_host = vr.host_vanish(g0, b0, verts, tets)
    assert np.array_equal(b1, b_host), f"{np.count_nonzero(b1 != b_host)} bitfield bytes differ from the host rule"
    if with_grid:
        assert np.array_equal(g1.view(np.uint32), g_host.view(np.uint32)), f"{np.count_nonzero(g1 != g_host)} grid cells differ from the host rule"
    assert n == int(changed_cells(g0, b0, g1, b1).sum())
    assert n > 0
    # a second call changes nothing
    assert r.cage_vanish(op_index, count=True, stream=stream) == 0
    g2, b2 = r.download_density_grid(want_grid=with_grid)
    assert np.array_equal(b2, b1) and (not with_grid or np.array_equal(g2.view(np.uint32), g1.view(np.uint32)))
    return g1, b1


@pytest.mark.parametrize("with_grid", [True, False], ids=["grid", "bitfield_only"])
@pytest.mark.parametrize("name", ["lattice4", "pulled", "coarse", "boundary", "flat"])
def test_vanish_after_set_edit_ops_matches_host_rule(scene, fresh, name, with_grid):
    model, occ = scene
    ov, dv, tets = vr.meshes(model)[name]
    affine = editing.AffineDuplication((0.5, 0.5, 0.5), (0.1, 0.1, 0.1), (0.1, 0.0, 0.0))
    op = as_operator(model, ov, dv, tets)
    fresh.set_edit_operators([affine.to_op(), op.to_op()])  # the cage is operator 1
    grid, bits = vr.inputs(seed=3)
    if with_grid:
        bits = fresh.upload_density_grid(grid)  # the context's bitfield is the grid's
    else:
        grid = None
        fresh.upload_occupancy(bits)
    _vanish_and_check(fresh, 1, op.vertices, op.tets, grid, bits, with_grid)


def test_cleared_cells_are_the_cells_with_a_lut_list(scene, fresh):
    """vanish and the renderer's tet lookup agree: the cells cleared are the cells whose operator list is non-empty."""
    model, _ = scene
    op = fx.make_cage(model, (0.45, 0.5, 0.55), (0.2, 0.15, 0.18), n_lattice=4)
    fresh.set_edit_operators([op.to_op()])
    fresh.upload_occupancy(np.full(abi.NSB_BITFIELD_BYTES, 0xFF, np.uint8))
    fresh.cage_vanish(0)
    _, bits = fresh.download_density_grid(want_grid=False)
    cleared = ~np.unpackbits(bits, bitorder="little").astype(bool)
    lut = fresh.cage_download(0, op.vertices.shape[0], op.tets.shape[0])["lut_offsets"]
    assert np.array_equal(cleared, np.diff(lut.astype(np.int64)) > 0)


@pytest.mark.parametrize("with_grid", [True, False], ids=["grid", "bitfield_only"])
def test_vanish_after_cage_deform_and_on_a_side_stream(scene, fresh, with_grid):
    import torch

    model, occ = scene
    op = fx.make_cage(model, (0.5, 0.62, 0.78), (0.17, 0.17, 0.17), n_lattice=4)
    fresh.set_edit_operators([op.to_op()])
    fresh.cage_attach_mvc(0, op.mvc)
    moved = op.cage_original.copy()
    moved[moved[:, 1] > op.cage_original[:, 1].mean()] += np.float32([0.03, 0.21, -0.05])
    op.cage_vertices = moved
    op.update_tet_mesh()        # host rebuild: op.vertices are what the device rebuild writes (test_gpu_edit_rebuild)
    grid, bits = vr.inputs(seed=4)
    if with_grid:
        bits = fresh.upload_density_grid(grid)
    else:
        grid = None
        fresh.upload_occupancy(bits)
    s = torch.cuda.Stream()
    fresh.cage_deform(0, op.cage_vertices, stream=s.cuda_stream)
    fresh.cage_vanish(0, stream=s.cuda_stream)   # stream-ordered behind the rebuild, no synchronisation
    s.synchronize()
    g1, b1 = fresh.download_density_grid(want_grid=with_grid)
    g_host, b_host = vr.host_vanish(grid, bits, op.vertices, op.tets)
    assert np.array_equal(b1, b_host)
    if with_grid:
        assert np.array_equal(g1.view(np.uint32), g_host.view(np.uint32))
    # and the counted path on the side stream: nothing left to clear
    assert fresh.cage_vanish(0, count=True, stream=s.cuda_stream) == 0


def test_vanish_argument_errors(scene, fresh):
    model, _ = scene
    lib, ctx = fresh.lib, fresh.ctx
    op = fx.make_cage(model, (0.5, 0.62, 0.78), (0.17, 0.17, 0.17))
    affine = editing.AffineDuplication((0.5, 0.5, 0.5), (0.1, 0.1, 0.1), (0.1, 0.0, 0.0))
    fresh.set_edit_operators([op.to_op(), affine.to_op()])
    n = C.c_uint64(7)
    assert lib.nsb_cage_vanish(ctx, 0, C.byref(n), None) == abi.NSB_ERR_STATE  # no occupancy yet
    assert n.value == 7
    fresh.upload_occupancy(np.full(abi.NSB_BITFIELD_BYTES, 0xFF, np.uint8))
    assert lib.nsb_cage_vanish(ctx, -1, None, None) == abi.NSB_ERR_INVALID
    assert lib.nsb_cage_vanish(ctx, 2, None, None) == abi.NSB_ERR_INVALID
    assert lib.nsb_cage_vanish(ctx, 1, None, None) == abi.NSB_ERR_INVALID  # affine
    assert lib.nsb_cage_vanish(None, 0, None, None) == abi.NSB_ERR_INVALID
    _, bits = fresh.download_density_grid(want_grid=False)
    assert (bits == 0xFF).all(), "a refused call changes nothing"
    assert lib.nsb_cage_vanish(ctx, 0, C.byref(n), None) == abi.NSB_OK and n.value > 0


@pytest.mark.parametrize("apply_operators", [True, False], ids=["operators", "no_operators"])
def test_frame_after_vanish_matches_oracle(scene, fresh, apply_operators):
    model, occ = scene
    ops = fx.e1(model)
    fresh.set_edit_operators([o.to_op() for o in ops])
    fresh.upload_occupancy(occ)
    frame = syn.make_frame(model, syn.fox_camera0(), 160, 90)
    frame.apply_operators = int(apply_operators)
    before = fresh.render(frame)[0].cpu().numpy()
    fresh.cage_vanish(0)
    after, depth = fresh.render(frame)
    after, depth = after.cpu().numpy(), depth.cpu().numpy()
    _, bits_host = vr.host_vanish(None, occ, ops[0].vertices, ops[0].tets)
    _, bits_dev = fresh.download_density_grid(want_grid=False)
    assert np.array_equal(bits_dev, bits_host)
    o_before = orc.Oracle(model.desc, model.params, occ, [op.to_op() for op in ops]).render(frame)[0]
    fb_o, depth_o, _, margin = orc.Oracle(model.desc, model.params, bits_host, [op.to_op() for op in ops]).render(frame, want_margin=True)
    _compare_frames(after, depth, fb_o, depth_o, margin)
    changed, changed_o = (after != before).any(-1), (fb_o != o_before).any(-1)
    print(f"\n{int(changed.sum())} of {changed.size} pixels changed ({int(changed_o.sum())} in the oracle)")
    assert changed.any()
    assert np.array_equal(changed, changed_o), f"{int((changed != changed_o).sum())} pixels change on one side only"


def test_grid_update_after_vanish_matches_oracle(scene, fresh):
    model, occ = scene
    ops = fx.e1(model)
    fresh.set_edit_operators([o.to_op() for o in ops])
    grid, _ = vr.inputs(seed=5)
    grid = np.abs(grid) * np.float32(0.02)  # a trained-looking grid: cells on both sides of the 0.01 threshold
    fresh.upload_density_grid(grid)
    fresh.cage_vanish(0)
    g_host, _ = vr.host_vanish(grid, np.zeros(abi.NSB_BITFIELD_BYTES, np.uint8), ops[0].vertices, ops[0].tets)
    rng = Pcg32(99)
    u = grid_params(400_000, 100_000, rng.copy(), ema_step=3, reset=False, apply_ops=False)
    g_cpu, b_cpu, mean = orc.Oracle(model.desc, model.params, occ).update_density_grid(u, g_host)
    fresh.update_density_grid(rng, 3, 400_000, 100_000, reset_grid=False, n_cascades=3, apply_operators=False)
    g_gpu, b_gpu = fresh.download_density_grid()
    exact, rel, nbytes = compare_grid_update(g_gpu, b_gpu, g_cpu, b_cpu, mean)
    print(f"\n{exact:.5f} of touched cells bit-equal, max |ln ratio| {rel:.3g}, {nbytes} bitfield bytes differ")
