"""nsb_update_density_grid over its parameter space, cell for cell.

Cell-exact check. The fused update (k_density_grid_update) and density-only nsb_density (k_inference<true, ACC16>) share
encode_to_a32 and tc::run_network, and each sample is one MMA row, so the raw fp16 density of a warped position is the same bits in
both kernels. The expected running grid is rebuilt on the host from the oracle's sample draw: nsb_density at the oracle's mapped
positions -> activation -> + the oracle's fp16 membrane residual (one __hadd: float64 sum rounded to fp16 once) -> * MIN_STEP ->
max-splat in uint order (np.maximum.at on the uint32 view, as testbed_nerf.cu:447-463) into the oracle's cells -> EMA. The device
grid must equal it bit for bit, and the device bitfield must equal the oracle's conversion of the device grid byte for byte.
NSB_ACT_NONE / RELU are exact on the host. Exponential and logistic use __expf / expf on the device and float64 here: a cell may
then take either fp16 rounding of a sample's activation when the activation lies within 2^-18 (relative) of an fp16 rounding
boundary, and only there; the number of cells that did is printed.

What it pins: the block boundaries of the sample remap in k_density_grid_update and the set of samples each launch draws (a lost,
duplicated or foreign sample changes a cell). What it cannot see: any bijective remap inside a 128^3 block passes by design, so the
warp locality of the remap is not tested here. It needs fixtures with at most one operator carrying membrane data, so that a
sample's residual is a single add.

Each case also runs test_gpu_grid_update._compare against the oracle's own MLP where the activation keeps every value positive."""
import contextlib

import numpy as np
import pytest

import edit_fixtures as fx
from nerfshop_b200 import abi
from nerfshop_b200.rng import Pcg32
from oracle import oracle as orc
from test_gpu_edit_rebuild import _drag
from test_gpu_grid_update import POLICIES, _compare
from test_grid_update_cpu import grid_params

pytestmark = pytest.mark.gpu

G = 128 ** 3
MIN_STEP = np.float32(1.73205080757) / np.float32(1024.0)
ACT_EPS = 2.0 ** -18  # __expf is within 2 + 1.2|x| fp32 ulps for the |x| < 12 that stay finite in fp16; 2^-18 is 32 ulps
ACTS = {"none": abi.NSB_ACT_NONE, "relu": abi.NSB_ACT_RELU, "logistic": abi.NSB_ACT_LOGISTIC, "exponential": abi.NSB_ACT_EXPONENTIAL}


@contextlib.contextmanager
def _restoring(renderer, occ, policy="f16"):
    """Runs under an accumulator policy on both sides and resets what the cases change on the shared renderer."""
    old = orc.set_mlp_policy(POLICIES[policy][1])
    try:
        renderer.set_mlp_accumulator(POLICIES[policy][0])
        yield
    finally:
        orc.set_mlp_policy(old)
        renderer.set_mlp_accumulator(abi.NSB_MLP_ACC_F16)
        renderer.reset_edit_operators()
        renderer.upload_occupancy(occ)


def _pattern_grid(untrained=False):
    """A running grid with ~15 % of cells just above NERF_MIN_OPTICAL_THICKNESS (the non-uniform draw's targets), ~7 % at 0.3 and,
    if asked, ~10 % untrained (negative) cells, in every cascade."""
    h = (np.arange(abi.NSB_GRID_CELLS, dtype=np.uint64) * np.uint64(2654435761)) % np.uint64(4096)
    g = np.zeros(abi.NSB_GRID_CELLS, np.float32)
    g[h < 600] = 0.0101
    g[(h >= 600) & (h < 900)] = 0.3
    if untrained:
        g[h >= 3700] = -1.0
    return g


def _params(n_uniform, n_nonuniform, rng, step=0, reset=False, n_cascades=3, act=abi.NSB_ACT_EXPONENTIAL, decay=0.95, aabb=None, ops=True):
    u = grid_params(n_uniform, n_nonuniform, rng, ema_step=step, reset=reset, n_cascades=n_cascades, apply_ops=ops)
    u.density_activation, u.decay = act, decay
    if aabb is not None:
        u.train_aabb_min[:], u.train_aabb_max[:] = aabb
    return u


def _update(renderer, u, rng, stream=0):
    """nsb_update_density_grid with the parameters of u; rng (u's state) is advanced like m_rng."""
    assert (rng.state, rng.inc) == (u.rng_state, u.rng_inc)
    renderer.update_density_grid(rng, u.ema_step, u.n_uniform_samples, u.n_nonuniform_samples, reset_grid=bool(u.reset_grid), n_cascades=u.n_cascades,
                                 decay=u.decay, train_aabb=(tuple(u.train_aabb_min), tuple(u.train_aabb_max)), density_activation=u.density_activation,
                                 apply_operators=bool(u.apply_operators), stream=stream)


def _fmaxf(a, b):
    """CUDA fmaxf: the non-NaN operand, +0 over -0."""
    return np.where(np.isnan(b) | (a > b) | ((a == b) & ~np.signbit(a)), a, b).astype(np.float32)


def _ema(prev, tmp, decay):
    """k_ema_grid (ema_grid_samples_nerf, testbed_nerf.cu:483-506): untrained cells stay, the rest take max(prev * decay, splat)."""
    return np.where(prev < 0, prev, _fmaxf(prev * np.float32(decay), tmp)).astype(np.float32)


def _expected_grids(renderer, u, prevs, samples, splats):
    """The running grid after one update, rebuilt from nsb_density at the oracle's mapped positions. One grid per activation
    rounding: [exact] for NONE / RELU, [low, host, high] for logistic / exponential. prevs: the grid before, one per rounding."""
    cells, residual = splats
    res = residual.view(np.float16).astype(np.float64)
    assert not np.isnan(res).any(), "at most one operator may add a membrane residual to a sample"
    coords = np.full((cells.size, 7), 0.5, np.float32)
    coords[:, :3] = samples[:, :3]
    coords[:, 3] = 0.0
    raw = renderer.density(coords)[0].view(np.float16).astype(np.float64)
    act = u.density_activation
    with np.errstate(over="ignore", invalid="ignore"):
        if act == abi.NSB_ACT_NONE:
            a, scales = raw, (1.0,)
        elif act == abi.NSB_ACT_RELU:
            a, scales = np.where(raw > 0, raw, 0.0), (1.0,)
        elif act == abi.NSB_ACT_LOGISTIC:
            a, scales = 1.0 / (1.0 + np.exp(-raw)), (1 - ACT_EPS, 1.0, 1 + ACT_EPS)
        else:
            a, scales = np.exp(raw), (1 - ACT_EPS, 1.0, 1 + ACT_EPS)
        out = []
        for s, prev in zip(scales, prevs if len(prevs) == len(scales) else [prevs[0]] * len(scales)):
            h = ((a * s).astype(np.float16).astype(np.float64) + res).astype(np.float16)  # __float2half_rn, then __hadd
            ot = h.astype(np.float32) * MIN_STEP
            tmp = np.zeros(abi.NSB_GRID_CELLS, np.uint32)
            np.maximum.at(tmp, cells, ot.view(np.uint32))
            out.append(_ema(prev, tmp.view(np.float32), u.decay))
    return out


def _check_exact(expected, g_gpu, b_gpu, label):
    """Device grid == the host rebuild cell for cell (the one-ulp activation allowance where `expected` has three roundings), and
    device bitfield == the oracle's conversion of the device grid. Returns the number of cells that took the allowance."""
    lo, mid, hi = expected[0], expected[len(expected) // 2], expected[-1]
    gu = g_gpu.view(np.uint32)
    same = (gu == lo.view(np.uint32)) | (gu == hi.view(np.uint32))
    between = (np.minimum(lo, hi) <= g_gpu) & (g_gpu <= np.maximum(lo, hi)) & (lo.view(np.uint32) != hi.view(np.uint32))
    bad = np.nonzero(~(same | between))[0]
    assert bad.size == 0, f"{label}: {bad.size} cells differ from the host rebuild, e.g. cells {bad[:6]}: device {g_gpu[bad[:6]]}, host {mid[bad[:6]]}"
    n_may = int((lo.view(np.uint32) != hi.view(np.uint32)).sum())
    n_took = int((gu != mid.view(np.uint32)).sum())
    assert n_may <= 0.03 * max(int((mid > 0).sum()), 1), f"{label}: {n_may} cells with two roundings"
    bits, _ = orc.density_grid_to_bitfield(g_gpu)
    assert np.array_equal(b_gpu, bits), f"{label}: {(b_gpu != bits).sum()} bitfield bytes differ from the oracle's conversion of the device grid"
    print(f"{label}: cell-exact; {n_took} cells took the one-ulp activation allowance ({n_may} could)")
    return n_took


def _case(renderer, o, u, rng, grid0, label, stream=0, tolerant=True):
    """One update from grid0 on the device and in the oracle: the cell-exact check, then (tolerant) _compare with the oracle's grid."""
    renderer.upload_density_grid(grid0)
    g_cpu, b_cpu, mean, samples, splats = o.update_density_grid(u, grid0, want_samples=True, want_splats=True)
    _update(renderer, u, rng.copy(), stream)
    g_gpu, b_gpu = renderer.download_density_grid()
    prev = np.zeros_like(grid0) if u.reset_grid else grid0
    _check_exact(_expected_grids(renderer, u, [prev], samples, splats), g_gpu, b_gpu, label)
    if tolerant:
        exact, rel, nbytes = _compare(g_gpu, b_gpu, g_cpu, b_cpu, mean)
        print(f"{label}: vs oracle MLP {exact:.5f} of touched cells bit-equal, max |ln ratio| {rel:.3g}, {nbytes} bitfield bytes differ")
    return g_gpu, b_gpu, splats[0]


def _oracle(model, occ, ops):
    return orc.Oracle(model.desc, model.params, occ, ops)


# ---- the sample remap: several blocks per launch, a non-uniform launch with a full block, a ragged tail ------------------------------
@pytest.mark.parametrize("policy", sorted(POLICIES))
def test_remap_several_blocks_and_a_nonuniform_block(scene, renderer, policy):
    """2 x 128^3 uniform + 128^3 non-uniform samples at ema_step 3 through E3: both launches contain full 128^3 blocks."""
    model, occ = scene
    ops = [op.to_op() for op in fx.e3(model)]
    with _restoring(renderer, occ, policy):
        renderer.set_edit_operators(ops)
        rng = Pcg32(2024)
        u = _params(2 * G, G, rng, step=3)
        _, _, cells = _case(renderer, _oracle(model, occ, ops), u, rng, _pattern_grid(), f"2x128^3 + 128^3 {policy}")
        assert np.unique(cells // G).tolist() == [0, 1, 2]


@pytest.mark.parametrize("policy", sorted(POLICIES))
def test_remap_ragged_tail(scene, renderer, policy):
    """128^3 + 12,345 uniform and 777 non-uniform samples at ema_step 5: one full block, then a tail the remap must leave alone;
    step * n_el is not a multiple of 2^21 and the total (2,110,274) is not a multiple of 128."""
    model, occ = scene
    ops = [op.to_op() for op in fx.e3(model)]
    with _restoring(renderer, occ, policy):
        renderer.set_edit_operators(ops)
        rng = Pcg32(77)
        u = _params(G + 12_345, 777, rng, step=5)
        assert (u.n_uniform_samples + u.n_nonuniform_samples) % 128 and (5 * u.n_uniform_samples) % (1 << 21)
        _case(renderer, _oracle(model, occ, ops), u, rng, _pattern_grid(), f"128^3+12345 / 777 {policy}")


# ---- cascades ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_cascades", [1, 2, 3, 4, 5])
def test_cascades(scene, renderer, n_cascades):
    model, occ = scene
    with _restoring(renderer, occ):
        rng = Pcg32(500 + n_cascades)
        u = _params(250_000, 50_000, rng, n_cascades=n_cascades, ops=False)
        grid0 = _pattern_grid()
        g_gpu, _, cells = _case(renderer, _oracle(model, occ, None), u, rng, grid0, f"{n_cascades} cascades")
        assert np.unique(cells // G).tolist() == list(range(n_cascades)), "every cascade is sampled"
        for k in range(n_cascades):  # and the device splatted into each of them
            assert (g_gpu[k * G:(k + 1) * G] > grid0[k * G:(k + 1) * G] * np.float32(0.95)).sum() > 1000, k


# ---- untrained cells -------------------------------------------------------------------------------------------------------------------
def test_untrained_cells(scene, renderer):
    """A grid with negative (untrained) cells: the draw steps over them, the EMA leaves them as they are, the mean counts them as 0."""
    model, occ = scene
    ops = [op.to_op() for op in fx.e1(model)]
    with _restoring(renderer, occ):
        renderer.set_edit_operators(ops)
        grid0 = _pattern_grid(untrained=True)
        neg = grid0 < 0
        rng = Pcg32(31)
        u = _params(300_000, 200_000, rng, step=2)
        g_gpu, b_gpu, cells = _case(renderer, _oracle(model, occ, ops), u, rng, grid0, "untrained cells")
        assert not neg[cells].any(), "no sample lands on an untrained cell"
        assert np.array_equal(g_gpu[neg].view(np.uint32), grid0[neg].view(np.uint32))
        # the threshold is min(0.01, mean of max(cell, 0)): with the negatives counted as themselves it would be below 0
        assert np.minimum(grid0[:G], 0).sum() / G < -0.05
        _, mean = orc.density_grid_to_bitfield(g_gpu)
        assert mean > 0.01


# ---- activations, decay, AABB, an empty update, a side stream --------------------------------------------------------------------------
@pytest.mark.parametrize("act", list(ACTS))
def test_density_activations(scene, renderer, act):
    """All four activations through E3 (membrane residuals included). With NONE, negative optical thickness wins the uint max
    (testbed_nerf.cu:443-462): pinned cell for cell."""
    model, occ = scene
    ops = [op.to_op() for op in fx.e3(model)]
    with _restoring(renderer, occ):
        renderer.set_edit_operators(ops)
        rng = Pcg32(900 + ACTS[act])
        u = _params(250_000, 50_000, rng, step=1, act=ACTS[act])
        # NONE / RELU can put a raw density on either side of 0 where the oracle's MLP and the device's differ by an ulp
        tolerant = ACTS[act] in (abi.NSB_ACT_LOGISTIC, abi.NSB_ACT_EXPONENTIAL)
        _case(renderer, _oracle(model, occ, ops), u, rng, _pattern_grid(), f"activation {act}", tolerant=tolerant)


def test_negative_optical_thickness_wins_the_splat(scene, renderer):
    """NSB_ACT_NONE on one cascade with 2 x 128^3 uniform samples: every cell is drawn twice, and in the cells where one sample is
    negative and the other positive the negative one wins the uint max (the reset grid then keeps 0, not the positive value)."""
    model, occ = scene
    with _restoring(renderer, occ):
        rng = Pcg32(17)
        u = _params(2 * G, 0, rng, reset=True, n_cascades=1, act=abi.NSB_ACT_NONE, ops=False)
        o = _oracle(model, occ, None)
        renderer.upload_density_grid(_pattern_grid())
        _, _, _, samples, splats = o.update_density_grid(u, _pattern_grid(), want_samples=True, want_splats=True)
        _update(renderer, u, rng.copy())
        g_gpu, b_gpu = renderer.download_density_grid()
        _check_exact(_expected_grids(renderer, u, [np.zeros(abi.NSB_GRID_CELLS, np.float32)], samples, splats), g_gpu, b_gpu, "negative wins")
        cells, h = splats[0], samples[:, 3]
        mixed = np.intersect1d(cells[h < 0], cells[h > 0])
        print(f"negative wins: {mixed.size} cells drew a negative and a positive sample")
        assert mixed.size > 100


@pytest.mark.parametrize("decay", [0.5, 1.0])
def test_decay(scene, renderer, decay):
    model, occ = scene
    with _restoring(renderer, occ):
        rng = Pcg32(41)
        u = _params(250_000, 50_000, rng, step=4, decay=decay, ops=False)
        _case(renderer, _oracle(model, occ, None), u, rng, _pattern_grid(), f"decay {decay}")


@pytest.mark.parametrize("aabb", [((0.0, 0.0, 0.0), (1.0, 1.0, 1.0)), ((-0.7, -1.2, -0.4), (1.9, 2.3, 1.6))], ids=["unit", "asymmetric"])
def test_train_aabb(scene, renderer, aabb):
    """Train AABBs other than the scene's own (-1.5..2.5 on every axis, which every other case uses), through E1."""
    model, occ = scene
    ops = [op.to_op() for op in fx.e1(model)]
    with _restoring(renderer, occ):
        renderer.set_edit_operators(ops)
        rng = Pcg32(43)
        u = _params(250_000, 50_000, rng, step=1, aabb=aabb)
        _case(renderer, _oracle(model, occ, ops), u, rng, _pattern_grid(), f"aabb {aabb}")


@pytest.mark.parametrize("reset", [False, True])
def test_empty_update(scene, renderer, reset):
    """n_total = 0: only the EMA with an empty splat (prev < 0 ? prev : max(prev * decay, 0)) and the bitfield rebuild run."""
    model, occ = scene
    with _restoring(renderer, occ):
        grid0 = _pattern_grid(untrained=True)
        renderer.upload_density_grid(grid0)
        rng = Pcg32(5)
        u = _params(0, 0, rng, reset=reset, decay=0.8)
        _update(renderer, u, rng)
        g_gpu, b_gpu = renderer.download_density_grid()
        expected = _ema(np.zeros_like(grid0) if reset else grid0, np.zeros_like(grid0), 0.8)
        assert np.array_equal(g_gpu.view(np.uint32), expected.view(np.uint32))
        assert np.array_equal(b_gpu, orc.density_grid_to_bitfield(expected)[0])
        assert reset or b_gpu.any()


def test_side_stream_matches_default_stream(scene, renderer):
    import torch

    model, occ = scene
    ops = [op.to_op() for op in fx.e3(model)]
    with _restoring(renderer, occ):
        renderer.set_edit_operators(ops)
        rng = Pcg32(61)
        u = _params(G + 4321, 100_000, rng, step=2)
        g_def, b_def, _ = _case(renderer, _oracle(model, occ, ops), u, rng, _pattern_grid(), "default stream")
        renderer.upload_density_grid(_pattern_grid())
        s = torch.cuda.Stream()
        r = rng.copy()
        _update(renderer, u, r, stream=s.cuda_stream)
        s.synchronize()
        g_side, b_side = renderer.download_density_grid()
        assert np.array_equal(g_side.view(np.uint32), g_def.view(np.uint32)) and np.array_equal(b_side, b_def)


def test_sample_count_bound_rejected_before_launch(scene, renderer):
    """Totals above NSB_GRID_UPDATE_MAX_SAMPLES (2^31, where the kernel's 32-bit grid-stride index could wrap) are refused before
    anything runs: the reset_grid of the refused call leaves the running grid as it was."""
    model, occ = scene
    with _restoring(renderer, occ):
        grid0 = _pattern_grid()
        renderer.upload_density_grid(grid0)
        for n_uniform, n_nonuniform in ((abi.NSB_GRID_UPDATE_MAX_SAMPLES, 1), (0xFFFFFFFF, 0xFFFFFFFF), (1 << 30, (1 << 31) + 1 - (1 << 30))):
            rng = Pcg32(1)
            with pytest.raises(abi.NsbError):
                renderer.update_density_grid(rng, 0, n_uniform, n_nonuniform, reset_grid=True)
            assert (rng.state, rng.inc) == (Pcg32(1).state, Pcg32(1).inc)
        g, _ = renderer.download_density_grid()
        assert np.array_equal(g.view(np.uint32), grid0.view(np.uint32))


# ---- the post-edit sequence -----------------------------------------------------------------------------------------------------------
def _post_edit_on_device(renderer, model, drag, membrane):
    op = fx.e1(model)[0]
    renderer.set_edit_operators([op.to_op()])
    renderer.cage_attach_mvc(0, op.mvc)
    if drag is not None:
        op.cage_vertices = _drag(op, drag)
        renderer.cage_deform(0, op.cage_vertices)  # the tet lookup is rebuilt on the device
    renderer.cage_set_membrane(0, op.mvc, *membrane, amplitude=1.0, apply=True)
    state = {"rng": Pcg32(11), "ema_step": 0, "max_cascade": 2}
    renderer.update_density_grid_nerf_render(state, 2, True)
    return state


def test_post_edit_sequence(scene, renderer):
    """set_edit_operators(E1) -> cage_attach_mvc -> cage_deform (a drag) -> cage_set_membrane -> update_density_grid_nerf_render
    (max_cascade 2, 2 iterations) on the device, against the same sequence on the host (update_tet_mesh, membrane_blend, the
    oracle's update with the host-rebuilt operator)."""
    model, occ = scene
    drag = (0.12, 0.05, -0.03)
    with _restoring(renderer, occ):
        base = fx.e1(model)[0]
        renderer.set_edit_operators([base.to_op()])
        d_in, s_in, _ = renderer.poisson_boundary(base.cage_original, is_inside=True, seed=5)
        dragged = _drag(base, drag)
        d_out, s_out, _ = renderer.poisson_boundary(dragged, is_inside=False, seed=6)
        membrane = (d_in, d_out, s_in, s_out)
        state = _post_edit_on_device(renderer, model, drag, membrane)
        g_gpu, b_gpu = renderer.download_density_grid()

        host = fx.e1(model)[0]
        host.cage_vertices = dragged
        host.update_tet_mesh()
        host.set_membrane(*orc.membrane_blend(host.mvc, *membrane), amplitude=1.0, apply=True)
        o = _oracle(model, occ, [host.to_op()])
        rng_o = Pcg32(11)
        g_cpu = np.zeros(abi.NSB_GRID_CELLS, np.float32)
        expected = [g_cpu]
        for it in range(2):
            u = _params(3 * G, 0, rng_o, step=it, reset=it == 0)
            g_cpu, b_cpu, mean, samples, splats = o.update_density_grid(u, g_cpu, want_samples=True, want_splats=True)
            expected = _expected_grids(renderer, u, expected, samples, splats)
            rng_o.advance(); rng_o.advance()
        assert (splats[1] != 0).sum() > 1000, "the membrane residual reaches the update"
        _check_exact(expected, g_gpu, b_gpu, "post-edit")
        exact, rel, nbytes = _compare(g_gpu, b_gpu, g_cpu, b_cpu, mean)
        print(f"post-edit: vs oracle MLP {exact:.5f} of touched cells bit-equal, max |ln ratio| {rel:.3g}, {nbytes} bitfield bytes differ")
        assert (state["rng"].state, state["rng"].inc) == (rng_o.state, rng_o.inc) and state["ema_step"] == 2

        # the drag moved occupancy: the same sequence without it gives another grid
        _post_edit_on_device(renderer, model, None, membrane)
        g_plain, _ = renderer.download_density_grid()
        assert (g_plain != g_gpu).sum() > 100
