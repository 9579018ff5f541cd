"""The CUDA path of this repository against the reference's OWN CUDA path, on the GPU.

oracle/_ref/libnerfshop_ref_cuda.so is the nvcc (sm_90a) build of the reference's sources — Testbed::render_nerf, NerfTracer::trace /
init_rays_from_camera and every kernel they launch, interpolate_tet, translate_in_box, compute_residual_poisson_kernel (oracle/ref_build.py,
oracle/ref_driver_cuda.cu) — with one substitution: tiny-cuda-nn's network (absent submodule) is this repository's nsb_inference. So what
these tests pin, against code the reference's authors wrote and the same compiler's FMA contraction, is everything AROUND the network:
ray generation, jitter, occupancy stepping, compaction/termination semantics, deformation, membrane blend, composite, shade.

  * ray / sample stream (t, dt, warped position): bit for bit;
  * frames without operators, including the 1920x1080 north-star configuration: bit for bit (L-inf = 0);
  * frames with operators: <= 1e-3 (measured 3e-5): interpolate_tet's barycentrics agree to 1 ulp only — ptxas fuses the mul/sub pairs of the
    reference kernel's cross products inconsistently (shared sub-expressions across the four same_side tests), which is not a contract.
The library is built where the reference's sources exist.
"""
import numpy as np
import pytest

from edit_fixtures import e1, e3
from nerfshop_b200 import abi, editing
from nerfshop_b200 import synthetic as syn
from ref_golden import ref

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not ref.cuda_usable("test_gpu_vs_ref_cuda"), reason="neither oracle/_ref nor stored reference results (tests/golden/ref/)")]

_a = 0.4
ROT = np.array([[np.cos(_a), -np.sin(_a), 0], [np.sin(_a), np.cos(_a), 0], [0, 0, 1]], np.float32)


def _affine():
    return editing.AffineDuplication((0.5, 0.5, 0.5), (0.12, 0.12, 0.12), (0.03, 0.0, -0.1), rotation=ROT, hide_original=True, correct_dir=True)


@pytest.fixture(scope="module")
def ref_cuda(scene):
    model, occ = scene
    rc = ref.RefCuda(occ)
    yield rc
    rc.close()


@pytest.mark.parametrize("cam_index,spp", [(17, 0), (63, 0), (99, 5)])
def test_sample_stream_bit_exact_vs_reference_kernels(scene, renderer, ref_cuda, cam_index, spp):
    model, occ = scene
    W, H, MS = 192, 108, 64
    f = syn.make_frame(model, syn.orbit_cameras(120)[cam_index], W, H, spp=spp)
    pix = np.random.default_rng(cam_index).choice(W * H, 6000, replace=False).astype(np.uint32)
    rec, idx, cnt = renderer.march_trace(f, pix, MS)
    rec_r, ray_r, cnt_r = ref_cuda.march_trace(f, pix, MS)
    frac = ref.fraction(cnt_r)  # a stored reference result keeps a seeded sample of the rays: compare on those
    rec, rec_r = ref.match(rec, rec_r)
    cnt, cnt_r = ref.match(cnt, cnt_r)
    assert np.array_equal(np.minimum(cnt, MS), cnt_r)
    amin, amax = np.array(list(f.train_aabb_min), np.float32), np.array(list(f.train_aabb_max), np.float32)
    valid = np.arange(MS)[None, :] < cnt_r[:, None]
    assert valid.sum() > 100_000 * frac
    t_after = (rec[..., 0] + rec[..., 1]).astype(np.float32)  # payload.t after `t += dt` (generate_next_nerf_network_inputs)
    assert np.array_equal(t_after[valid], rec_r[..., 7][valid])
    wp = ((rec[..., 2:5] - amin) / (amax - amin)).astype(np.float32)  # warp_position(pos, train_aabb): one sub, one div per component
    assert np.array_equal(wp[valid], rec_r[..., 0:3][valid])
    min_step = np.float32(np.float32(1.73205080757) / np.float32(1024.0))
    wdt = ((rec[..., 1] - min_step) / (min_step * np.float32(16.0) - min_step)).astype(np.float32)  # warp_dt
    assert np.array_equal(wdt[valid], rec_r[..., 3][valid])


@pytest.mark.parametrize("cam_index,mode", [(17, abi.NSB_RENDER_SHADE), (63, abi.NSB_RENDER_SHADE), (5, abi.NSB_RENDER_DEPTH), (40, abi.NSB_RENDER_COST), (77, abi.NSB_RENDER_POSITIONS)])
def test_frame_identical_to_reference_render_nerf(scene, renderer, ref_cuda, cam_index, mode):
    import torch

    model, occ = scene
    f = syn.make_frame(model, syn.orbit_cameras(120)[cam_index], 320, 180)
    f.render_mode = mode
    fb, depth = renderer.render(f)
    st = renderer.stats()
    fb_r, depth_r, info = ref_cuda.render(f, renderer)
    torch.cuda.synchronize()
    assert st.n_samples > 100_000 and info["n_calls"] % 2 == 0 and info["n_inferred"] >= 2 * st.n_samples  # the reference infers every batch twice
    fb, fb_r = ref.match(fb, fb_r)  # a stored reference frame keeps a seeded sample of its rows
    depth, depth_r = ref.match(depth, depth_r)
    assert torch.equal(fb, fb_r)
    assert torch.equal(depth, depth_r)


def test_north_star_1080p_frames_identical_to_reference_render_nerf(scene, renderer, ref_cuda):
    """configs[0]/[1]: nerf/fox camera C0 and orbit cameras at 1920x1080, no edits: RGBA and depth equal the reference's CUDA path bit for bit."""
    import torch

    model, occ = scene
    cams = [syn.fox_camera0()] + [syn.orbit_cameras(120)[i] for i in (0, 45, 90)]
    for cam in cams:
        f = syn.make_frame(model, cam, 1920, 1080)
        fb, depth = renderer.render(f)
        fb_r, depth_r, info = ref_cuda.render(f, renderer)
        torch.cuda.synchronize()
        assert (fb[..., 3] > 0).float().mean().item() > 0.2
        fb, fb_r = ref.match(fb, fb_r)
        depth, depth_r = ref.match(depth, depth_r)
        err = (fb - fb_r).abs().max().item()
        assert err == 0.0, err
        assert torch.equal(depth, depth_r)


def _edit_scenes(model):
    yield "E1 (configs[2]: one cage)", [c.to_op() for c in e1(model)], 1
    ops = [c.to_op() for c in e3(model)] + [_affine().to_op()]
    yield "E3 + affine, poisson_target on (configs[3])", ops, 1
    yield "E3 + affine, poisson_target off", ops, 0


def test_edit_operator_kernels_vs_reference(scene, renderer):
    model, occ = scene
    ops = [c.to_op() for c in e3(model)] + [_affine().to_op()]
    renderer.set_edit_operators(ops)
    rc = ref.RefCuda(occ, ops)
    try:
        rng = np.random.default_rng(3)
        n = 400_000
        c = np.zeros((n, 7), np.float32)
        c[:, :3] = rng.uniform(0.38, 0.64, (n, 3))
        d = rng.standard_normal((n, 3)).astype(np.float32)
        c[:, 4:] = (d / np.linalg.norm(d, axis=1, keepdims=True) + 1) * 0.5
        cn, mn = renderer.map_rays(c)
        cr0, mr = rc.map_rays(c)
        frac = ref.fraction(cr0)  # a stored reference result keeps a seeded sample of the coordinates: compare on those
        cn, cr = ref.match(cn, cr0)
        mn, mr = ref.match(mn, mr)
        cs, _ = ref.match(c, cr0)
        moved = (cr[:, :3] != cs[:, :3]).any(axis=1)
        assert moved.sum() > 20_000 * frac and mr.sum() > 10_000 * frac
        assert np.array_equal(mn, mr)                                   # empty mask: identical
        assert np.array_equal((cn[:, :3] != cs[:, :3]).any(axis=1), moved)  # same samples found a tet / a box
        assert np.array_equal(cn[:, 3:], cr[:, 3:])                     # dt and mapped direction: identical
        assert np.abs(cn[:, :3] - cr[:, :3]).max() <= 2.0 ** -23        # mapped position: 1 ulp (see module docstring)
        sh, od, rd = renderer.poisson_residuals(c)
        sh_r, od_r, rd_r = rc.poisson_residuals(c)
        frac = ref.fraction(od_r)
        sh, sh_r = ref.match(sh, sh_r)
        od, od_r = ref.match(od, od_r)
        rd, rd_r = ref.match(rd, rd_r)
        assert (od_r != 0).sum() > 5000 * frac and np.array_equal(od != 0, od_r != 0)
        assert np.allclose(od, od_r, rtol=1e-6, atol=1e-5) and np.allclose(rd, rd_r, rtol=1e-6, atol=1e-5) and np.allclose(sh, sh_r, rtol=1e-6, atol=1e-6)
    finally:
        rc.close()
        renderer.set_edit_operators([])


def test_edited_1080p_frames_vs_reference_render_nerf(scene, renderer):
    """configs[2] and configs[3] at 1920x1080 against the reference's CUDA path (map_rays / compute_poisson_full_residuals / membrane composite)."""
    import torch

    model, occ = scene
    cam = syn.orbit_cameras(120)[17]
    for name, ops, target in _edit_scenes(model):
        renderer.set_edit_operators(ops)
        rc = ref.RefCuda(occ, ops)
        try:
            f = syn.make_frame(model, cam, 1920, 1080)
            f.apply_operators, f.poisson_target = 1, target
            fb, depth = renderer.render(f)
            st = renderer.stats()
            fb_r, depth_r, _ = rc.render(f, renderer)
            f0 = syn.make_frame(model, cam, 1920, 1080)
            fb0, _ = renderer.render(f0)
            torch.cuda.synchronize()
            changed = ((fb - fb0).abs().amax(-1) > 1e-3).sum().item()
            fb, fb_r = ref.match(fb, fb_r)  # a stored reference frame keeps a seeded sample of its rows
            err = (fb - fb_r).abs().amax(-1)
            print(f"\n{name}: L-inf {err.max().item():.3e}, pixels > 1e-4: {(err > 1e-4).sum().item()}, edit changed {changed} pixels, old-density samples {st.n_old_samples}")
            assert changed > 5000
            assert err.max().item() <= 1e-3
            assert (err > 1e-4).sum().item() <= 50
        finally:
            rc.close()
            renderer.set_edit_operators([])
