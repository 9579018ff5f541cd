"""§8(f)-1 on the GPU: nsb_cage_deform rebuilds a dragged cage's tet mesh on the device (MVC interpolation, boxes, per-tet
rotations, the 5 x 128^3 CSR tet lookup) — against the host implementation of the same reference rules
(nsb_host_geometry.cpp <- cage.cu:39-55, tet_mesh.cu:13-20,38-74,369-667), which tests/test_editing_cpu.py pins.
Vertices, boxes and the CSR are bit-identical (the device repeats the host's non-contracted fp32 arithmetic); rotations come
from a double-precision Newton iteration and agree to float rounding."""
import numpy as np
import pytest

import edit_fixtures as fx
from nerfshop_b200 import synthetic as syn
from oracle import oracle as orc
from test_gpu_parity import _compare_frames

pytestmark = pytest.mark.gpu


def _drag(op, pull):
    moved = op.cage_original.copy()
    moved[moved[:, 0] > op.cage_original[:, 0].mean()] += np.asarray(pull, np.float32)
    return moved


def _check_against_host(renderer, op_index, op):
    got = renderer.cage_download(op_index, op.vertices.shape[0], op.tets.shape[0], rotations=op.use_local_rotations)
    assert np.array_equal(got["vertices"].view(np.uint32), op.vertices.view(np.uint32)), "MVC interpolation must be bit-exact"
    host_op, _ = op.to_op()
    boxes = np.array(list(host_op.bbox_min) + list(host_op.bbox_max) + list(host_op.warped_bbox_min) + list(host_op.warped_bbox_max), np.float32)
    assert np.array_equal(got["boxes"].view(np.uint32), boxes.view(np.uint32))
    assert np.array_equal(got["lut_offsets"], op.lut_offsets), f"{(got['lut_offsets'] != op.lut_offsets).sum()} CSR offsets differ"
    assert np.array_equal(got["lut_idx"], op.lut_idx)
    if op.use_local_rotations:
        assert np.abs(got["rotations"] - op.rotations).max() < 2e-6
    return got


def test_cage_deform_matches_host_rebuild(scene, renderer):
    model, occ = scene
    try:
        ops = fx.e3(model)
        renderer.set_edit_operators([o.to_op() for o in ops])
        for i, o in enumerate(ops):
            renderer.cage_attach_mvc(i, o.mvc)
        # three successive drags of operator 0 (the last one large: the list outgrows the uploaded array), one of operator 2
        for pull in ((0.02, 0.0, 0.01), (0.12, 0.05, -0.03), (0.45, 0.2, 0.1)):
            ops[0].cage_vertices = _drag(ops[0], pull)
            ops[0].update_tet_mesh()                       # host rebuild
            renderer.cage_deform(0, ops[0].cage_vertices)  # device rebuild
            got = _check_against_host(renderer, 0, ops[0])
        assert got["lut_idx"].size > 0
        ops[2].cage_vertices = _drag(ops[2], (0.0, 0.06, 0.0))
        ops[2].update_tet_mesh()
        renderer.cage_deform(2, ops[2].cage_vertices)
        _check_against_host(renderer, 2, ops[2])
        _check_against_host(renderer, 0, ops[0])  # untouched by the other operator's rebuild
        # and the renderer marches the rebuilt operators: frame == oracle frame with the host-rebuilt operators
        o = orc.Oracle(model.desc, model.params, occ, [op.to_op() for op in ops])
        frame = syn.make_frame(model, syn.fox_camera0(), 160, 90)
        frame.apply_operators = 1
        fb, depth = renderer.render(frame)
        fb_o, depth_o, st_o, margin = o.render(frame, want_margin=True)
        _compare_frames(fb.cpu().numpy(), depth.cpu().numpy(), fb_o, depth_o, margin)
        assert renderer.stats().n_samples == st_o.n_samples
    finally:
        renderer.reset_edit_operators()


def test_cage_deform_long_cell_lists(scene, renderer):
    """10,368 tets: the coarse-cascade cells list every tet (> 8192 entries -> the global-scratch bitonic path of k_tet_sort_long)."""
    model, _ = scene
    try:
        # a small cage that sits inside ONE cascade-4 cell ([0.5,0.625]^2 x [0.75,0.875]): that cell lists all 10,368 tets
        op = fx.make_cage(model, (0.56, 0.56, 0.81), (0.05, 0.05, 0.05), pull=(0.004, 0.0, 0.0), n_lattice=12)
        renderer.set_edit_operators([op.to_op()])
        renderer.cage_attach_mvc(0, op.mvc)
        op.cage_vertices = _drag(op, (0.008, -0.002, 0.003))
        op.update_tet_mesh()
        renderer.cage_deform(0, op.cage_vertices)
        got = _check_against_host(renderer, 0, op)
        assert np.diff(got["lut_offsets"].astype(np.int64)).max() > 8192
    finally:
        renderer.reset_edit_operators()


def test_cage_deform_argument_errors(scene, renderer):
    from nerfshop_b200 import abi, editing

    model, _ = scene
    try:
        op = fx.e1(model)[0]
        aff = editing.AffineDuplication((0.6, 0.55, 0.5), (0.05, 0.05, 0.05), (0.04, 0.02, 0.0))
        renderer.set_edit_operators([op.to_op(), aff.to_op()])
        with pytest.raises(abi.NsbError):
            renderer.cage_deform(0, op.cage_vertices)          # MVC not attached
        with pytest.raises(abi.NsbError):
            renderer.cage_attach_mvc(1, op.mvc)                # not a cage
        with pytest.raises(abi.NsbError):
            renderer.cage_attach_mvc(2, op.mvc)                # out of range
        renderer.cage_attach_mvc(0, op.mvc)
        with pytest.raises(abi.NsbError):
            renderer.cage_deform(0, op.cage_vertices[:-1])     # wrong cage size
    finally:
        renderer.reset_edit_operators()
