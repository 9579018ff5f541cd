"""§8(f)-2 on the GPU: nsb_update_density_grid (fused draw -> map_positions -> hash encode + density MLP -> activate ->
membrane residual -> max-splat, then EMA merge and bitfield rebuild) against the oracle's restatement of
Testbed::update_density_grid_nerf_operator (testbed_nerf.cu:3533-3639).

Tolerances: cell selection, sample positions, operator mapping and the splat/EMA/bitfield logic are integer/pinned-fp32 work and
must agree exactly; the density value goes through the fp16 MLP (wgmma fp32 accumulation vs the oracle's wide accumulation:
raw outputs within a few fp16 ulps, test_gpu_parity) and __expf, so a cell's value may differ by the fp16 spacing of the raw
output: |ln(gpu/cpu)| <= 4 ulp_fp16(raw) <= 4 * 2^-7 for |raw| < 8. Bitfield bytes may differ only where a cell of that byte sits
within that tolerance of the threshold."""
import numpy as np
import pytest

import edit_fixtures as fx
from nerfshop_b200 import abi
from nerfshop_b200.rng import Pcg32
from oracle import oracle as orc
from test_grid_update_cpu import grid_params

pytestmark = pytest.mark.gpu

RTOL = 4 * 2.0 ** -7


def _compare(g_gpu, b_gpu, g_cpu, b_cpu, mean_cpu):
    assert np.array_equal(g_gpu > 0, g_cpu > 0), "the set of touched cells must be identical (integer cell selection)"
    nz = g_cpu > 0
    exact = (g_gpu[nz] == g_cpu[nz]).mean()
    rel = np.abs(np.log(g_gpu[nz].astype(np.float64) / g_cpu[nz].astype(np.float64)))
    assert exact > 0.98, f"only {exact:.4f} of touched cells bit-equal"
    assert rel.max() <= RTOL, f"max |ln ratio| {rel.max():.4g}"
    thresh = min(0.01, mean_cpu)
    near = np.abs(np.log(np.maximum(g_cpu, 1e-30) / thresh)) <= RTOL
    # level-0..4 bytes straight from the grid: allowed to differ only next to the threshold
    diff_bytes = np.nonzero(b_gpu != b_cpu)[0]
    direct = np.packbits(near.reshape(-1, 8), axis=1, bitorder="little").reshape(-1) != 0
    # a differing bit of cascade k may propagate into cascades k+1.. through bitfield_max_pool; accept those only if some
    # near-threshold cell exists at all, and bound their number
    if diff_bytes.size:
        assert near.any()
        assert diff_bytes.size <= 8 * int(direct.sum()), (diff_bytes.size, int(direct.sum()))
    return exact, rel.max(), diff_bytes.size


def test_grid_update_no_operators(scene, renderer):
    model, occ = scene
    o = orc.Oracle(model.desc, model.params, occ)
    rng = Pcg32(1337)
    rng_o = rng.copy()
    g_cpu = np.zeros(abi.NSB_GRID_CELLS, np.float32)
    state = {"rng": rng, "ema_step": 0}
    try:
        for step, (nu, nn, reset) in enumerate([(600_000, 0, True), (300_000, 200_000, False)]):
            u = grid_params(nu, nn, rng_o, ema_step=step, reset=reset)
            g_cpu, b_cpu, mean = o.update_density_grid(u, g_cpu)
            rng_o.advance(); rng_o.advance()
            renderer.update_density_grid(state["rng"], state["ema_step"], nu, nn, reset_grid=reset, n_cascades=3)
            state["ema_step"] += 1
            g_gpu, b_gpu = renderer.download_density_grid()
            exact, rel, nbytes = _compare(g_gpu, b_gpu, g_cpu, b_cpu, mean)
            print(f"step {step}: {exact:.5f} of touched cells bit-equal, max |ln ratio| {rel:.3g}, {nbytes} bitfield bytes differ")
            g_cpu = g_gpu.copy()  # continue both from the same state so the second step's cell selection stays comparable
        assert (state["rng"].state, state["rng"].inc) == (rng_o.state, rng_o.inc)
    finally:
        renderer.upload_occupancy(occ)


@pytest.mark.parametrize("fixture", ["e1", "e3"])
def test_grid_update_through_operators(scene, renderer, fixture):
    model, occ = scene
    ops = [op.to_op() for op in getattr(fx, fixture)(model)]
    o = orc.Oracle(model.desc, model.params, occ, ops)
    renderer.set_edit_operators(ops)
    try:
        rng = Pcg32(99)
        u = grid_params(128 ** 3, 0, rng, n_cascades=1)  # every cascade-0 cell index is visited (the index is a bijection mod 128^3)
        g_cpu, b_cpu, mean = o.update_density_grid(u, np.zeros(abi.NSB_GRID_CELLS, np.float32))
        renderer.update_density_grid(rng.copy(), 0, 128 ** 3, 0, reset_grid=True, n_cascades=1)
        g_gpu, b_gpu = renderer.download_density_grid()
        exact, rel, nbytes = _compare(g_gpu, b_gpu, g_cpu, b_cpu, mean)
        print(f"{fixture}: {exact:.5f} bit-equal, max |ln ratio| {rel:.3g}, {nbytes} bitfield bytes differ")
        # and the operators did change the grid
        g_plain, _, _ = orc.Oracle(model.desc, model.params, occ).update_density_grid(u, np.zeros(abi.NSB_GRID_CELLS, np.float32))
        assert (g_plain != g_cpu).sum() > 100
    finally:
        renderer.reset_edit_operators()
        renderer.upload_occupancy(occ)


def test_render_marches_the_updated_bitfield(scene, renderer):
    """After an update the renderer must march the rebuilt bitfield: render == oracle render with the downloaded bitfield."""
    from nerfshop_b200 import synthetic as syn
    from test_gpu_parity import _compare_frames

    model, occ = scene
    try:
        st = {"rng": Pcg32(3), "ema_step": 0, "max_cascade": 2}
        renderer.update_density_grid_nerf_render(st, 1, True)
        assert st["ema_step"] == 1
        _, bits = renderer.download_density_grid(want_grid=False)
        assert bits.any() and not np.array_equal(bits, occ)
        frame = syn.make_frame(model, syn.fox_camera0(), 160, 90)
        fb, depth = renderer.render(frame)
        o = orc.Oracle(model.desc, model.params, bits)
        fb_o, depth_o, stats_o, margin = o.render(frame, want_margin=True)
        _compare_frames(fb.cpu().numpy(), depth.cpu().numpy(), fb_o, depth_o, margin)
        assert renderer.stats().n_samples == stats_o.n_samples
    finally:
        renderer.upload_occupancy(occ)
