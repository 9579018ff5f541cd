"""§8(f)-4 on the GPU: nsb_poisson_boundary (directions on the host, inference on wgmma, activation + SH9 fit on the device) and
nsb_cage_set_membrane (the gamma-coordinate blend into the operator's device arrays) against the oracle.
Tolerances: colours/densities pass the fp16 MLP (raw outputs within a few fp16 ulps) and expf -> density within 4 ulp_fp16(raw)
relative, SH coefficients (means of ~100 colours in (0,1) times |Y| <= 1.1, scaled by 4pi) within 2e-3. The blend is pinned fp32 on
identical inputs -> bit-exact."""
import numpy as np
import pytest

import edit_fixtures as fx
from nerfshop_b200 import synthetic as syn
from oracle import oracle as orc
from test_gpu_parity import _compare_frames

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("inside", [False, True])
def test_poisson_boundary_matches_oracle(scene, renderer, oracle, inside):
    model, occ = scene
    op = fx.e1(model)[0]
    pts = np.concatenate([op.cage_original if inside else op.cage_vertices, np.array([[2.3, 2.3, 2.3]], np.float32)])
    dens, shs, p = renderer.poisson_boundary(pts, is_inside=inside, seed=21)
    dens_o, shs_o = oracle.poisson_boundary(pts, p)
    assert np.array_equal(dens == 0, dens_o == 0)
    nz = dens_o > 0
    assert np.abs(np.log(dens[nz] / dens_o[nz])).max() <= 4 * 2.0 ** -7
    assert np.abs(shs - shs_o).max() < 2e-3, np.abs(shs - shs_o).max()
    # (the float values themselves differ in the last place: __expf on the device, libm expf in the oracle)
    assert np.median(np.abs(np.log(dens[nz] / dens_o[nz]))) < 1e-5
    if inside:
        assert dens[-1] == 0.0


def test_cage_set_membrane_bit_exact_and_rendered(scene, renderer):
    model, occ = scene
    try:
        op = fx.e1(model)[0]
        renderer.set_edit_operators([op.to_op()])
        # GrowingSelection::interpolate_poisson_boundary: inside values at the canonical cage, outside values at the deformed one
        d_in, s_in, _ = renderer.poisson_boundary(op.cage_original, is_inside=True, seed=5)
        d_out, s_out, _ = renderer.poisson_boundary(op.cage_vertices, is_inside=False, seed=6)
        gamma = op.mvc  # mvc_gamma = 1: the gamma coordinates are the MVC weights (cage.cu:25)
        b_shs, b_od, b_rd = renderer.cage_set_membrane(0, gamma, d_in, d_out, s_in, s_out, amplitude=1.0, apply=True)
        o_shs, o_od, o_rd = orc.membrane_blend(gamma, d_in, d_out, s_in, s_out)
        assert np.array_equal(b_shs.view(np.uint32), o_shs.view(np.uint32))
        assert np.array_equal(b_od.view(np.uint32), o_od.view(np.uint32)) and np.array_equal(b_rd.view(np.uint32), o_rd.view(np.uint32))
        assert np.abs(b_shs).max() > 1e-3
        # the renderer now blends with these arrays: same frame as the oracle given the same arrays through the upload path
        op.set_membrane(o_shs, o_od, o_rd, amplitude=1.0, apply=True)
        o = orc.Oracle(model.desc, model.params, occ, [op.to_op()])
        frame = syn.make_frame(model, syn.fox_camera0(), 160, 90, apply_operators=True)
        fb, depth = renderer.render(frame)
        fb_o, depth_o, st_o, margin = o.render(frame, want_margin=True)
        _compare_frames(fb.cpu().numpy(), depth.cpu().numpy(), fb_o, depth_o, margin)
        assert renderer.stats().n_samples == st_o.n_samples
        # and it differs from the same edit without the membrane
        renderer.set_edit_operators([fx.e1(model)[0].to_op()])
        fb_plain, _ = renderer.render(frame)
        assert np.abs(fb_plain.cpu().numpy() - fb.cpu().numpy()).max() > 1e-3
    finally:
        renderer.reset_edit_operators()
