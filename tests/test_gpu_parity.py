"""GPU parity tests proper: the CUDA path (through the C ABI) against the CPU oracle on the same seeded
inputs and against the committed golden vectors. Bars (DESIGN.md §3):
  * occupancy march (sample t / dt / position / mip / cell index): BIT-EXACT
  * hash-grid encoding (fp16 features): BIT-EXACT
  * fused MLP outputs: fp16 values within 2 fp16 ulps + 1e-3 (tensor-core fp32 accumulation order is not pinned)
  * framebuffer RGBA: L-inf <= 1e-3 (north_star), excluding pixels the oracle flags as sitting on the
    early-termination threshold within float noise (their branch may legitimately flip); depth <= 1e-3 relative.
"""
import os

import numpy as np
import pytest

from conftest import random_coords
from nerfshop_b200 import abi, synthetic as syn

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "synthetic_fox.npz")
RGBA_TOL = 1e-3
MARGIN_EPS = 2e-5  # |A - 0.99| below this: termination branch is within accumulated float noise


def _half(a):
    return a.view(np.float16).astype(np.float32)


def _ulp_close(got_u16, ref_u16, ulps=2, atol=1e-3):
    g, r = _half(got_u16), _half(ref_u16)
    tol = ulps * np.maximum(np.abs(r), 2.0 ** -14) * 2.0 ** -10 + atol
    bad = np.abs(g - r) > tol
    return bad


def test_library_loaded_is_the_cuda_extension(renderer):
    # the product path has no fallback: the context exists only if libnerfshop_b200.so loaded and found an sm_90 device
    assert renderer.ctx
    with open("/proc/self/maps") as fh:
        assert "libnerfshop_b200.so" in fh.read()


def test_march_bit_exact(scene, oracle, renderer):
    model, _ = scene
    for cam, (w, h) in ((syn.fox_camera0(), (160, 90)), (syn.orbit_cameras(120)[40], (96, 54))):
        f = syn.make_frame(model, cam, w, h)
        pix = np.arange(0, w * h, 5, dtype=np.uint32)
        rec_o, idx_o, cnt_o = oracle.march_trace(f, pix, 160)
        rec_g, idx_g, cnt_g = renderer.march_trace(f, pix, 160)
        assert (cnt_o == cnt_g).all(), f"sample counts differ on {(cnt_o != cnt_g).sum()} rays"
        assert cnt_o.sum() > 10000
        assert (idx_o == idx_g).all()
        assert (rec_o.view(np.uint32) == rec_g.view(np.uint32)).all(), "t/dt/pos bits differ"


def test_march_bit_exact_with_jitter_and_subpixel(scene, oracle, renderer):
    model, _ = scene
    f = syn.make_frame(model, syn.orbit_cameras(120)[77], 128, 72, spp=5)
    pix = np.arange(0, 128 * 72, 3, dtype=np.uint32)
    rec_o, idx_o, cnt_o = oracle.march_trace(f, pix, 64)
    rec_g, idx_g, cnt_g = renderer.march_trace(f, pix, 64)
    assert (cnt_o == cnt_g).all() and (idx_o == idx_g).all()
    assert (rec_o.view(np.uint32) == rec_g.view(np.uint32)).all()


def test_encode_bit_exact(oracle, renderer):
    coords = random_coords(4099, seed=11)  # ragged: not a multiple of 128
    coords[:7, :3] = [[0, 0, 0], [1, 1, 1], [0.5, 0.5, 0.5], [1, 0, 0.25], [0.999999, 0.5, 1e-7], [0.25, 1, 1], [0, 1, 0]]  # box corners/faces
    ref = oracle.encode(coords)
    got = renderer.encode(coords)
    assert got.shape == ref.shape
    assert (got == ref).all(), f"{(got != ref).sum()} of {got.size} fp16 features differ"


def test_density_and_inference_vs_oracle(oracle, renderer):
    coords = random_coords(1000, seed=12)  # ragged tail (1000 = 7*128 + 104)
    ref_d = oracle.inference(coords, density_only=True)
    got_d = renderer.density(coords)
    bad = _ulp_close(got_d, ref_d)
    assert bad.mean() < 1e-3, f"density MLP: {bad.sum()} of {bad.size} outputs off by more than 2 ulp"
    exact = (got_d == ref_d).mean()
    assert exact > 0.97, f"only {exact:.3f} of density outputs bit-equal"
    ref = oracle.inference(coords)
    got = renderer.inference(coords)
    assert (got[3] == got_d[0]).all()  # extract_density: row 3 is the density MLP's out[0]
    bad = _ulp_close(got[:4], ref[:4], ulps=4, atol=2e-3)
    assert bad.mean() < 2e-3, f"rgb MLP: {bad.sum()} of {bad.size} outputs outside tolerance"
    assert np.abs(_half(got[:3]) - _half(ref[:3])).max() < 0.05


def test_inference_empty_and_single(oracle, renderer):
    assert renderer.inference(np.zeros((0, 7), np.float32)).shape == (16, 0)
    c = random_coords(1, seed=5)
    got, ref = renderer.inference(c), oracle.inference(c)
    assert not _ulp_close(got[:4], ref[:4], ulps=4, atol=2e-3).any()


def test_inference_matches_golden(renderer):
    g = np.load(GOLDEN)
    got = renderer.inference(g["coords"])
    assert (renderer.encode(g["coords"]) == g["encode"]).all()
    assert _ulp_close(got[:4], g["inference"][:4], ulps=4, atol=2e-3).mean() < 2e-3


def _compare_frames(fb_g, depth_g, fb_o, depth_o, margin):
    """L-inf RGBA <= 1e-3 on every pixel, except that a pixel whose accumulated alpha came within float noise of
    the early-termination threshold may legitimately take the other branch — at most a handful per frame."""
    diff = np.abs(fb_g - fb_o).max(axis=-1)
    bad = diff > RGBA_TOL
    ambiguous = margin <= MARGIN_EPS
    assert not (bad & ~ambiguous).any(), f"L-inf RGBA {diff[~ambiguous].max():.2e} > {RGBA_TOL} on {(bad & ~ambiguous).sum()} unambiguous pixels"
    assert (bad & ambiguous).sum() <= max(2, diff.size // 20000), f"{(bad & ambiguous).sum()} threshold pixels flipped"
    same_hit = (depth_o < 1e9) == (depth_g < 1e9)
    assert same_hit.mean() > 0.9995
    hit = (depth_o < 1e9) & (depth_g < 1e9) & ~bad
    if hit.any():
        derr = np.abs(depth_g[hit] - depth_o[hit])
        assert np.quantile(derr, 0.999) <= 1e-3 * np.abs(depth_o[hit]).max() + 1e-4  # depth = position of the max-weight sample (ties can flip)
    return float(diff.max())


def test_render_matches_golden(scene, renderer):
    model, _ = scene
    g = np.load(GOLDEN)
    for name, cam in (("fox0", syn.fox_camera0()), ("orbit17", syn.orbit_cameras(120)[17])):
        f = syn.make_frame(model, cam, 96, 54)
        fb, depth = renderer.render(f)
        st = renderer.stats()
        fb, depth = fb.cpu().numpy(), depth.cpu().numpy()
        _compare_frames(fb, depth, g[f"{name}_rgba"], g[f"{name}_depth"], g[f"{name}_margin"])
        n_rays, n_alive, n_hit, n_samples = (int(v) for v in g[f"{name}_stats"])
        assert st.n_rays == n_rays and st.n_rays_alive == n_alive
        assert abs(int(st.n_hit) - n_hit) <= 2
        assert abs(int(st.n_samples) - n_samples) <= max(50, n_samples // 2000)  # a flipped termination adds/removes a few samples


def test_render_vs_oracle_ragged_resolution(scene, oracle, renderer):
    """Resolution that is not a multiple of the 16x8 tile, non-zero spp index, background over-blend."""
    model, _ = scene
    import torch

    f = syn.make_frame(model, syn.orbit_cameras(120)[95], 203, 117, spp=2)
    bg = np.zeros((117, 203, 4), np.float32)
    bg[..., 2] = 0.25
    bg[..., 3] = 1.0
    fb_o, depth_o, st_o, margin = oracle.render(f, background=bg, want_margin=True)
    fb = torch.from_numpy(bg.copy()).cuda()
    fb, depth = renderer.render(f, fb=fb)
    _compare_frames(fb.cpu().numpy(), depth.cpu().numpy(), fb_o, depth_o, margin)
    st = renderer.stats()
    assert st.n_rays == 203 * 117 and st.n_rays_alive == st_o.n_rays_alive


def test_render_modes_vs_oracle(scene, oracle, renderer):
    model, _ = scene
    for mode in (abi.NSB_RENDER_AO, abi.NSB_RENDER_POSITIONS, abi.NSB_RENDER_DEPTH, abi.NSB_RENDER_STEPSIZE, abi.NSB_RENDER_COST):
        f = syn.make_frame(model, syn.orbit_cameras(120)[3], 64, 36, render_mode=mode)
        fb_o, depth_o, _, margin = oracle.render(f, want_margin=True)
        fb, depth = renderer.render(f)
        d = np.abs(fb.cpu().numpy() - fb_o).max(-1)
        tol = 2e-2 if mode == abi.NSB_RENDER_COST else 2e-3  # cost = step count / 128: one flipped step is 1/128
        assert (d > tol).sum() <= 2, f"mode {mode}: {d.max()}"


def test_render_host_entry_point(scene, oracle, renderer):
    model, _ = scene
    f = syn.make_frame(model, syn.fox_camera0(), 80, 45)
    fb_h, depth_h = renderer.render_to_cpu(f)
    fb_d, depth_d = renderer.render(f)
    assert np.array_equal(fb_h, fb_d.cpu().numpy()) and np.array_equal(depth_h, depth_d.cpu().numpy())  # deterministic per pixel


def test_tile_partition_union_equals_single(scene, renderer):
    """Image-plane partition: rendering tiles t % world == rank for every rank reproduces the single-GPU frame
    bit for bit (per-pixel results do not depend on which CTA/GPU marches the ray)."""
    import torch

    model, _ = scene
    cam = syn.orbit_cameras(120)[60]
    W, H = 176, 99
    full, dfull = renderer.render(syn.make_frame(model, cam, W, H))
    total_rays = 0
    for world in (2, 3):
        acc = torch.zeros_like(full)
        dacc = torch.zeros_like(dfull)
        for rank in range(world):
            fb, depth = renderer.render(syn.make_frame(model, cam, W, H, rank=rank, world=world))
            total_rays += renderer.stats().n_rays
            n_tiles = renderer.tiles_for_rank(W, H, rank, world)
            packed = torch.zeros((n_tiles * 128, 4), dtype=torch.float32, device="cuda")
            pdepth = torch.zeros(n_tiles * 128, dtype=torch.float32, device="cuda")
            renderer.pack_tiles(fb, depth, rank, world, packed, pdepth)
            renderer.unpack_tiles(packed, pdepth, rank, world, acc, dacc)
        torch.cuda.synchronize()
        assert torch.equal(acc, full) and torch.equal(dacc, dfull)
    assert total_rays == 2 * W * H
    # the N > 1 frame of bench.py / parallel.gather_framebuffer: RGBA + depth of every rank in ONE gathered buffer, ONE unpack launch
    for world in (2, 4):
        n = renderer.tiles_for_rank(W, H, 0, world) * 128  # pixels per shard (rank 0 owns the most tiles)
        gathered = torch.zeros((world, 5 * n), dtype=torch.float32, device="cuda")
        for rank in range(world):
            fb, depth = renderer.render(syn.make_frame(model, cam, W, H, rank=rank, world=world))
            renderer.pack_tiles(fb, depth, rank, world, gathered[rank, : 4 * n].view(n, 4), gathered[rank, 4 * n:])
        own, down = renderer.render(syn.make_frame(model, cam, W, H, rank=1, world=world))  # rank 1's view: its own tiles are in place already
        renderer.unpack_gathered(gathered[:, : 4 * n], gathered[:, 4 * n:], gathered.stride(0), 1, world, own, down)
        torch.cuda.synchronize()
        assert torch.equal(own, full) and torch.equal(down, dfull)


def test_full_size_properties(scene, renderer):
    """BASELINE size (1920x1080): size-independent properties instead of a CPU comparison —
    determinism (two renders are bit-identical), ray/sample accounting, alpha in [0,1], finite values,
    and agreement of a 1080p crop-by-partition with the full frame."""
    import torch

    model, _ = scene
    f = syn.make_frame(model, syn.orbit_cameras(120)[17], 1920, 1080)
    fb1, d1 = renderer.render(f)
    st1 = renderer.stats()
    fb2, d2 = renderer.render(f)
    st2 = renderer.stats()
    assert torch.equal(fb1, fb2) and torch.equal(d1, d2)
    assert st1.n_rays == 1920 * 1080 and st1.n_samples == st2.n_samples and st1.n_hit == st2.n_hit
    assert torch.isfinite(fb1).all()
    a = fb1[..., 3]
    assert float(a.min()) >= 0.0 and float(a.max()) <= 1.0 + 1e-6
    assert int((a > 0.001).sum()) == st1.n_hit  # every shaded ray wrote its pixel (black background)
    assert st1.n_samples > 20 * st1.n_hit * 0.2


def test_async_host_frames_equal_the_synchronous_ones(scene, renderer):
    """nsb_render_host_async / nsb_host_frame_wait: five frames through two slots in flight equal nsb_render_host's, tickets count up, and a bad
    ticket is an error."""
    import torch

    model, _ = scene
    cams = syn.orbit_cameras(120)
    W, H = 320, 180
    frames = [syn.make_frame(model, cams[(11 * k) % 120], W, H) for k in range(5)]
    want = [tuple(a.copy() for a in renderer.render_to_cpu(f)) for f in frames]
    host = [(torch.zeros((H, W, 4)).pin_memory(), torch.zeros((H, W)).pin_memory()) for _ in range(5)]
    tickets = [renderer.render_to_cpu_async(f, *host[k]) for k, f in enumerate(frames)]
    assert tickets == list(range(tickets[0], tickets[0] + 5))
    for k in (4, 3, 0, 1, 2):
        renderer.wait_host_frame(tickets[k])
    for k in range(5):
        assert np.array_equal(host[k][0].numpy(), want[k][0]) and np.array_equal(host[k][1].numpy(), want[k][1])
    assert renderer.lib.nsb_host_frame_wait(renderer.ctx, tickets[-1] + 1) == abi.NSB_ERR_INVALID


def test_no_model_is_an_error(built_lib):
    import ctypes as C

    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    lib = abi.load_library()
    ctx = C.c_void_p()
    assert lib.nsb_create(0, C.byref(ctx)) == abi.NSB_OK
    f = abi.NsbFrame()
    buf = torch.zeros(16, device="cuda")
    assert lib.nsb_render(ctx, C.byref(f), buf.data_ptr(), buf.data_ptr(), None) == abi.NSB_ERR_STATE
    assert b"nsb_upload_model" in lib.nsb_last_error()
    lib.nsb_destroy(ctx)


def test_unit_cube_scene_constant_step(renderer, built_lib):
    """aabb_scale = 1 (the reference's synthetic-Lego shape): cone angle 0 -> constant dt = sqrt(3)/1024, one cascade,
    per_level_scale 1.3819 -> FIVE dense levels, so the level pair (4,5) is mixed dense/hashed (the generic index path)."""
    from nerfshop_b200.renderer import NerfRenderer
    from oracle import oracle as orc

    model = syn.make_model(seed=7, aabb_scale=1)
    occ = syn.make_occupancy(model)
    assert abs(model.desc.per_level_scale - 1.3819) < 1e-3
    o = orc.Oracle(model.desc, model.params, occ)
    r = NerfRenderer(0)
    try:
        r.upload_model(model.desc, model.params)
        r.upload_occupancy(occ)
        coords = random_coords(2000, seed=21)
        assert (r.encode(coords) == o.encode(coords)).all()
        cam = syn.look_at((0.5, 0.6, 1.6))
        f = syn.make_frame(model, cam, 112, 63)
        assert f.cone_angle_constant == 0.0
        pix = np.arange(0, 112 * 63, 3, dtype=np.uint32)
        rec_o, idx_o, cnt_o = o.march_trace(f, pix, 256)
        rec_g, idx_g, cnt_g = r.march_trace(f, pix, 256)
        assert (cnt_o == cnt_g).all() and (idx_o == idx_g).all() and (rec_o.view(np.uint32) == rec_g.view(np.uint32)).all()
        assert cnt_o.max() > 20 and (idx_o[..., 0] == 0).all()  # a single cascade
        fb_o, depth_o, st_o, margin = o.render(f, want_margin=True)
        fb, depth = r.render(f)
        _compare_frames(fb.cpu().numpy(), depth.cpu().numpy(), fb_o, depth_o, margin)
        assert r.stats().n_samples == st_o.n_samples
    finally:
        r.close()


def test_empty_and_tiny_frames(scene, oracle, renderer):
    """No ray enters the AABB (camera outside, looking away): nothing is queued, the framebuffer keeps its content and depth is
    1e10 everywhere; 1x1 / 3x2 / 16x8 (exactly one tile) frames match the oracle."""
    import torch

    model, _ = scene
    away = syn.look_at((6.0, 6.0, 6.0), target=(12.0, 12.0, 12.0))
    f = syn.make_frame(model, away, 64, 36)
    bg = torch.full((36, 64, 4), 0.125, device="cuda")
    fb, depth = renderer.render(f, fb=bg.clone())
    st = renderer.stats()
    assert torch.equal(fb, bg) and bool((depth == 1e10).all())
    assert st.n_rays == 64 * 36 and st.n_rays_alive == 0 and st.n_samples == 0 and st.n_hit == 0
    for (w, h) in ((1, 1), (3, 2), (16, 8)):
        f = syn.make_frame(model, syn.fox_camera0(), w, h)
        fb_o, depth_o, st_o, margin = oracle.render(f, want_margin=True)
        fb, depth = renderer.render(f)
        assert np.abs(fb.cpu().numpy() - fb_o).max() <= RGBA_TOL or (margin <= MARGIN_EPS).any()
        assert renderer.stats().n_samples == st_o.n_samples
