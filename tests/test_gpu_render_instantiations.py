"""Every instantiation of the fused renderer, at frame sizes where its ray slots refill.

k_render_fused<OPS, ACC16, IN_RANGE> has six instantiations: operators or not, fp16 or fp32 MLP accumulators
(nsb_set_mlp_accumulator), and the in-range grid index (render AABB inside the train AABB, no operators) or the exact one. A CTA holds
7, 6 or 5 tiles of 128 ray slots (fp16 / fp32 / operators), one CTA per SM. Each warp claims 32 consecutive queue entries and claims
again once it is down to REFILL_THR = 2 live rays, so a slot takes more than one ray only in frames with more queued rays than the grid
has slots. nsb_debug_counters' last counter is the number of tiles that ran; a frame counts as in the refill regime here when
n_rays_alive > 2 x tiles run x 128.

  * the host picks the instantiation: tiles run of a 36-tile frame whose every pixel is queued;
  * frames without operators, both policies, train and wider render AABBs, 1920x1080: bit for bit against the reference's own
    render_nerf (oracle/ref_build.py), whose network is this repository's nsb_inference under the context's policy, on a schedule of its own;
  * frames with operators: inert operators (over empty occupancy) change no bit of a frame; an affine duplication alone is bit for bit
    the reference's frame; E1 under fp32 accumulators within the bar of the edited 1080p frames (test_gpu_vs_ref_cuda.py);
  * per-ray results do not depend on the schedule: the image-plane partitions of a 1080p frame reassemble it bit for bit, and its ray,
    hit and sample counts add up, in all six instantiations;
  * queue boundaries: frames of S - 1, S, S + 1, S + 33 and 2S + 1 queued rays (S = the slots of a full grid, from the device's SM
    count) equal the union of their partitions.
Every case that changes the policy, the operators or the occupancy of the module's context restores them.
"""
import contextlib

import numpy as np
import pytest

from edit_fixtures import e1, e3
from nerfshop_b200 import abi, editing
from nerfshop_b200 import synthetic as syn
from ref_golden import ref
from test_gpu_encoding_domain import _occupancy_with_outer_cascades
from test_gpu_vs_ref_cuda import _affine

pytestmark = pytest.mark.gpu

POLICIES = {"f16": abi.NSB_MLP_ACC_F16, "f32": abi.NSB_MLP_ACC_F32}
W, H = 1920, 1080
PAST_AABB = ((-2.5, -2.5, -2.5), (3.5, 4.0, 4.5))  # around the fox train AABB [-1.5, 2.5]^3 (as test_gpu_encoding_domain.py)
needs_ref = pytest.mark.skipif(not ref.cuda_usable("test_gpu_render_instantiations"), reason="neither oracle/_ref nor stored reference results (tests/golden/ref/)")


def _tiles_per_cta(ops: bool, policy: str) -> int:
    return 5 if ops else 7 if policy == "f16" else 6


@pytest.fixture(scope="module")
def r(scene, built_lib):
    """A context of this module's own: the frames below switch policy, operators and occupancy."""
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nerfshop_b200.renderer import NerfRenderer

    model, occ = scene
    rr = NerfRenderer(0)
    rr.upload_model(model.desc, model.params)
    rr.upload_occupancy(occ)
    yield rr
    rr.close()


@pytest.fixture(scope="module")
def sms(r):
    import torch

    return torch.cuda.get_device_properties(r.device).multi_processor_count


@contextlib.contextmanager
def _state(r, scene, policy="f16", ops=None, occ=None):
    model, occ0 = scene
    try:
        r.set_mlp_accumulator(POLICIES[policy])
        if ops:
            r.set_edit_operators(ops)
        if occ is not None:
            r.upload_occupancy(occ)
        yield
    finally:
        r.set_mlp_accumulator(abi.NSB_MLP_ACC_F16)
        r.set_edit_operators([])
        r.upload_occupancy(occ0)


def _frame(model, cam, w=W, h=H, aabb=None, **kw):
    f = syn.make_frame(model, cam, w, h, **kw)
    if aabb is not None:
        for a in range(3):
            f.render_aabb_min[a], f.render_aabb_max[a] = aabb[0][a], aabb[1][a]
    return f


def _render(r, f):
    """(fb, depth, stats, tiles run)."""
    fb, depth = r.render(f)
    st = r.stats()
    return fb, depth, st, r.debug_counters()["tiles"]


def _regime(name, st, tiles):
    ratio = st.n_rays_alive / (tiles * 128)
    print(f"\n{name}: n_rays_alive {st.n_rays_alive}, tiles run {tiles}, rays per slot {ratio:.2f}")
    return ratio


def _full_occupancy():
    return np.full(abi.NSB_BITFIELD_BYTES, 255, np.uint8)


def _inert_ops(model):
    """A cage and an affine duplication (source and destination box) inside 0.375-wide cubes of space where the scene's occupancy is
    empty on every cascade: no marched sample reaches them, so they map nothing."""
    cage = editing.lattice_cage(model, (1.92, 1.77, 1.61), (0.1, 0.1, 0.1), pull=(0.03, 0.0, 0.0))
    w = lambda p: tuple((np.float32(v) + np.float32(1.5)) / np.float32(4.0) for v in p)  # world -> warped (train AABB [-1.5, 2.5]^3)
    src, dst = np.array(w((-1.27, 1.23, -0.64))), np.array(w((-1.30, 1.23, 0.02)))
    affine = editing.AffineDuplication(src, (0.05, 0.05, 0.05), dst - src, hide_original=True, correct_dir=True)
    return [cage.to_op(), affine.to_op()]


def _e3_affine(model):
    return [c.to_op() for c in e3(model)] + [_affine().to_op()]


# ---- 1. the host's choice --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ops", [False, True], ids=["no_ops", "ops"])
@pytest.mark.parametrize("policy", sorted(POLICIES))
def test_host_picks_the_instantiation(r, scene, sms, policy, ops):
    """96x48 = 36 image tiles, every pixel queued (full occupancy, camera inside the AABB): ceil(36 / T) CTAs of T tiles run, and a CTA
    runs only if its first slot has a queue entry, so the tiles run are 42 (fp16), 36 (fp32) or 40 (operators, either policy)."""
    model, _ = scene
    assert sms * 5 >= 36
    with _state(r, scene, policy, _inert_ops(model) if ops else None, _full_occupancy()):
        f = _frame(model, syn.orbit_cameras(120)[30], 96, 48, apply_operators=ops)
        _, _, st, tiles = _render(r, f)
    assert st.n_rays_alive == 96 * 48
    assert tiles == (40 if ops else 42 if policy == "f16" else 36)
    assert _regime(f"96x48 {policy} ops={ops}", st, tiles) <= 2  # one ray per slot at most: below the refill regime


# ---- 2. frames without operators against the reference's render_nerf -------------------------------------------------------
@needs_ref
@pytest.mark.parametrize("policy", sorted(POLICIES))
def test_no_operator_frames_identical_to_reference_render_nerf(r, scene, sms, policy):
    """fp32: the render AABB equal to the train AABB (<false,false,true>) and past it (<false,false,false>); fp16: past it
    (<false,true,false>; fp16 in range is test_north_star_1080p_frames_identical_to_reference_render_nerf) and one NSB_RENDER_COST frame,
    whose value counts the steps of its ray (reset per slot on refill). Past the train AABB, occupancy in cascades 3-4 reaches the
    outer box. The call order is fixed: stored reference frames carry no array inputs."""
    import torch

    model, occ = scene
    occ2 = _occupancy_with_outer_cascades(occ)
    cams = [("fox C0", syn.fox_camera0()), ("orbit 45", syn.orbit_cameras(120)[45])]
    cases = []  # (name, bitfield, render AABB, mode)
    if policy == "f32":
        cases += [(f"{n}, train AABB", occ, None, abi.NSB_RENDER_SHADE, cam) for n, cam in cams]
    cases += [(f"{n}, past the train AABB", occ2, PAST_AABB, abi.NSB_RENDER_SHADE, cam) for n, cam in cams]
    if policy == "f16":
        cases.append(("orbit 45, cost", occ, None, abi.NSB_RENDER_COST, cams[1][1]))
    T = _tiles_per_cta(False, policy)
    for name, bits, aabb, mode, cam in cases:
        rc = ref.RefCuda(bits)
        try:
            with _state(r, scene, policy, occ=bits):
                f = _frame(model, cam, aabb=aabb, render_mode=mode)
                fb, depth, st, tiles = _render(r, f)
                fb_r, depth_r, _ = rc.render(f, r)
                torch.cuda.synchronize()
        finally:
            rc.close()
        assert tiles == sms * T and _regime(f"{policy} {name}", st, tiles) > 2
        assert (fb[..., 3] > 0).float().mean().item() > 0.2
        fb, fb_r = ref.match(fb, fb_r)  # a stored reference frame keeps a seeded sample of its rows
        depth, depth_r = ref.match(depth, depth_r)
        err = (fb - fb_r).abs().max().item()
        assert err == 0.0, f"{policy} {name}: L-inf {err:.3e} on {int(((fb - fb_r).abs().amax(-1) > 0).sum())} pixels"
        assert torch.equal(depth, depth_r), f"{policy} {name}: depth differs"


# ---- 3. frames with operators (5 tiles per CTA) ----------------------------------------------------------------------------
@pytest.mark.parametrize("policy", sorted(POLICIES))
def test_inert_operators_change_no_bit_of_the_frame(r, scene, sms, policy):
    """Operators over empty occupancy: <true, *, false> renders the same frame as the no-operator instantiation (<false, *, true>),
    bit for bit, and counts the same rays, hits and samples. The premise first: nsb_map_rays leaves the frame's marched samples as they
    are and empties none."""
    import torch

    model, _ = scene
    cam = syn.orbit_cameras(120)[17]
    with _state(r, scene, policy, _inert_ops(model)):
        f = _frame(model, cam)
        pix = np.arange(0, W * H, 13, dtype=np.uint32)
        rec, _, cnt = r.march_trace(f, pix, 64)
        live = np.arange(64)[None, :] < np.minimum(cnt, 64)[:, None]
        pos = rec[live][:, 2:5]
        assert pos.shape[0] > 100_000
        c = np.zeros((pos.shape[0], 7), np.float32)
        c[:, :3] = (pos - np.float32(-1.5)) / np.float32(4.0)
        c[:, 3] = rec[live][:, 1]
        d = pos.astype(np.float64) - np.asarray(cam[:, 3], np.float64)
        c[:, 4:] = (d / np.linalg.norm(d, axis=1, keepdims=True) + 1) * 0.5
        mapped, mask = r.map_rays(c)
        assert not mask.any()
        np.testing.assert_array_equal(mapped[:, :3].view(np.uint32), c[:, :3].view(np.uint32))
        fb0, depth0, st0, tiles0 = _render(r, _frame(model, cam))
        fb1, depth1, st1, tiles1 = _render(r, _frame(model, cam, apply_operators=True))
        torch.cuda.synchronize()
    assert tiles0 == sms * _tiles_per_cta(False, policy) and tiles1 == sms * 5
    assert _regime(f"{policy} inert operators", st1, tiles1) > 2
    assert torch.equal(fb1, fb0) and torch.equal(depth1, depth0)
    assert (st1.n_rays, st1.n_rays_alive, st1.n_hit, st1.n_samples) == (st0.n_rays, st0.n_rays_alive, st0.n_hit, st0.n_samples)


@needs_ref
def test_affine_only_frames_identical_to_reference_render_nerf(r, scene, sms):
    """An affine duplication alone (no tets: nothing goes through interpolate_tet), both policies: bit for bit the reference's frame."""
    import torch

    model, occ = scene
    cam = syn.orbit_cameras(120)[17]
    ops = [_affine().to_op()]
    for policy in sorted(POLICIES):
        rc = ref.RefCuda(occ, ops)
        try:
            with _state(r, scene, policy, ops):
                f = _frame(model, cam, apply_operators=True)
                fb, depth, st, tiles = _render(r, f)
                fb_r, depth_r, _ = rc.render(f, r)
                fb0, _ = r.render(_frame(model, cam))
                torch.cuda.synchronize()
        finally:
            rc.close()
        assert tiles == sms * 5 and _regime(f"{policy} affine only", st, tiles) > 2
        assert ((fb - fb0).abs().amax(-1) > 1e-3).sum().item() > 5000  # the duplication is visible
        fb, fb_r = ref.match(fb, fb_r)
        depth, depth_r = ref.match(depth, depth_r)
        err = (fb - fb_r).abs().amax(-1)
        assert err.max().item() == 0.0, f"{policy}: L-inf {err.max().item():.3e}, {(err > 0).sum().item()} pixels differ"
        assert torch.equal(depth, depth_r), f"{policy}: depth differs"


@needs_ref
def test_e1_fp32_frame_vs_reference_render_nerf(r, scene, sms):
    """configs[2] (E1, one cage) under fp32 accumulators at the bar of test_edited_1080p_frames_vs_reference_render_nerf."""
    import torch

    model, occ = scene
    cam = syn.orbit_cameras(120)[17]
    ops = [c.to_op() for c in e1(model)]
    rc = ref.RefCuda(occ, ops)
    try:
        with _state(r, scene, "f32", ops):
            f = _frame(model, cam, apply_operators=True, poisson_target=True)
            fb, depth, st, tiles = _render(r, f)
            fb_r, _, _ = rc.render(f, r)
            torch.cuda.synchronize()
    finally:
        rc.close()
    assert tiles == sms * 5 and _regime("f32 E1", st, tiles) > 2
    fb, fb_r = ref.match(fb, fb_r)
    err = (fb - fb_r).abs().amax(-1)
    print(f"f32 E1: L-inf {err.max().item():.3e}, pixels > 1e-4: {(err > 1e-4).sum().item()}")
    assert err.max().item() <= 1e-3
    assert (err > 1e-4).sum().item() <= 50


# ---- 4. per-ray results do not depend on the schedule ----------------------------------------------------------------------
def _union_of_partitions(r, make, full, dfull, world):
    """Renders rank 0..world-1 of the frame make(rank, world) and reassembles them; returns (fb, depth, summed stats, per-rank (stats, tiles))."""
    import torch

    acc, dacc = torch.zeros_like(full), torch.zeros_like(dfull)
    sums = np.zeros(5, np.uint64)
    ranks = []
    h, w = full.shape[0], full.shape[1]
    for rank in range(world):
        fb, depth, st, tiles = _render(r, make(rank, world))
        sums += np.array([st.n_rays, st.n_rays_alive, st.n_hit, st.n_samples, st.n_old_samples], np.uint64)
        ranks.append((st, tiles))
        n_tiles = r.tiles_for_rank(w, h, rank, world)
        packed = torch.zeros((n_tiles * 128, 4), dtype=torch.float32, device=full.device)
        pdepth = torch.zeros(n_tiles * 128, dtype=torch.float32, device=full.device)
        r.pack_tiles(fb, depth, rank, world, packed, pdepth)
        r.unpack_tiles(packed, pdepth, rank, world, acc, dacc)
    torch.cuda.synchronize()
    return acc, dacc, sums, ranks


def _counts(st):
    return np.array([st.n_rays, st.n_rays_alive, st.n_hit, st.n_samples, st.n_old_samples], np.uint64)


INSTANTIATIONS = {  # name: (policy, render AABB past the train AABB, operators); the kernel the host picks for it
    "f16-in_range": ("f16", False, False),   # <false, true, true>
    "f32-in_range": ("f32", False, False),   # <false, false, true>
    "f16-exact_index": ("f16", True, False),  # <false, true, false>
    "f32-exact_index": ("f32", True, False),  # <false, false, false>
    "f16-ops": ("f16", False, True),          # <true, true, false>
    "f32-ops": ("f32", False, True),          # <true, false, false>
}


@pytest.mark.parametrize("name", list(INSTANTIATIONS))
def test_partitions_reassemble_the_1080p_frame(r, scene, sms, name):
    """The 1080p frame and the union of its world = 2, 3 and 7 image-plane partitions: RGBA and depth bit-identical, and the ray, hit
    and sample counts of the ranks add up to the frame's. With operators the frame is E3 + affine with the membrane's poisson_target on,
    so the old-density samples add up too."""
    import torch

    model, occ = scene
    policy, past, ops_on = INSTANTIATIONS[name]
    cam = syn.orbit_cameras(120)[17]
    ops = _e3_affine(model) if ops_on else None
    bits = _occupancy_with_outer_cascades(occ) if past else None
    make = lambda rank=0, world=1: _frame(model, cam, aabb=PAST_AABB if past else None, rank=rank, world=world, apply_operators=ops_on,
                                          poisson_target=ops_on)
    with _state(r, scene, policy, ops, bits):
        full, dfull, st, tiles = _render(r, make())
        torch.cuda.synchronize()
        assert tiles == sms * _tiles_per_cta(ops_on, policy) and _regime(name, st, tiles) > 2
        assert st.n_rays == W * H and st.n_samples > 0 and (st.n_old_samples > 0) == ops_on
        for world in (2, 3, 7):
            acc, dacc, sums, _ = _union_of_partitions(r, make, full, dfull, world)
            assert torch.equal(acc, full), f"{name} world {world}: {int(((acc - full).abs().amax(-1) > 0).sum())} pixels differ"
            assert torch.equal(dacc, dfull), f"{name} world {world}: depth differs"
            np.testing.assert_array_equal(sums, _counts(st), err_msg=f"{name} world {world}: n_rays, n_rays_alive, n_hit, n_samples, n_old_samples")


# ---- 5. queue boundaries ---------------------------------------------------------------------------------------------------
def _shape_for(n, min_tiles):
    """W x H = n with at least min_tiles 16x8 image tiles: the largest H <= sqrt(n) that divides n and keeps enough tiles."""
    for h in range(int(np.sqrt(n)), 0, -1):
        if n % h == 0 and -(-(n // h) // 16) * -(-h // 8) >= min_tiles:
            return n // h, h
    raise AssertionError(n)


@pytest.mark.parametrize("kind", ["f16", "f32", "ops"])
def test_queue_boundaries_equal_the_union_of_partitions(r, scene, sms, kind):
    """Every pixel queued (full occupancy, camera inside the AABB), S = the ray slots of a full grid (SMs x T x 128): frames of S - 1, S,
    S + 1, S + 33 and 2S + 1 queued rays, each with at least SMs x T image tiles so that the grid is full. Each equals the union of its
    world = 3 partitions, which queue at most 2 rays per slot that runs."""
    import torch

    model, _ = scene
    ops_on = kind == "ops"
    policy = "f16" if ops_on else kind
    T = _tiles_per_cta(ops_on, policy)
    S = sms * T * 128
    cam = syn.orbit_cameras(120)[70]
    with _state(r, scene, policy, [c.to_op() for c in e1(model)] if ops_on else None, _full_occupancy()):
        for n in (S - 1, S, S + 1, S + 33, 2 * S + 1):
            w, h = _shape_for(n, sms * T)

            def make(rank=0, world=1):
                f = _frame(model, cam, w, h, rank=rank, world=world, apply_operators=ops_on)
                f.focal_length[0] = f.focal_length[1] = float(max(w, h))
                return f

            full, dfull, st, tiles = _render(r, make())
            torch.cuda.synchronize()
            assert st.n_rays_alive == n and tiles == sms * T, (n, st.n_rays_alive, tiles)
            ratio = _regime(f"{kind} {w}x{h} (S{n - S:+d})", st, tiles)
            assert (ratio > 2) == (n == 2 * S + 1)
            acc, dacc, sums, ranks = _union_of_partitions(r, make, full, dfull, 3)
            assert torch.equal(acc, full), f"{kind} n = S{n - S:+d}: {int(((acc - full).abs().amax(-1) > 0).sum())} pixels differ"
            assert torch.equal(dacc, dfull), f"{kind} n = S{n - S:+d}: depth differs"
            np.testing.assert_array_equal(sums, _counts(st))
            assert all(s.n_rays_alive <= 2 * t * 128 for s, t in ranks)
