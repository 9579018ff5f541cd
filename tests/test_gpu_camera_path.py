"""Camera paths and video frames on the GPU (ABI 8): nsb_render_accumulate is bit for bit the chain of nsb_render -> nsb_accumulate ->
nsb_tonemap it replaces, on plain, fp32-accumulator, edited (cage + membrane), depth-of-field, environment-map and lens-distortion frames;
nsb_frame_to_rgba8 equals scripts/run.py's numpy formula (write_image, transcribed below); render_video writes the frames the device
computed, deterministically, without touching the context's state."""
import ctypes as C
import os

import numpy as np
import pytest

import edit_fixtures as fx
from nerfshop_b200 import abi
from nerfshop_b200 import camera_path as cp
from nerfshop_b200 import synthetic as syn
from png_decode import decode_png
from test_frame_extras_cpu import CASES

pytestmark = pytest.mark.gpu

W, H = 160, 90


def _path() -> cp.CameraPath:
    cams = syn.orbit_cameras(120)
    kfs = [cp.CameraKeyframe.from_matrix(cams[i], slice=0.0, scale=1.0 + 0.1 * k, fov=50.625 - 4.0 * k, dof=0.0)
           for k, i in enumerate((14, 17, 21))]
    return cp.CameraPath(kfs)


def _sub_frames(base, spp, t0=0.2, t1=0.3, spp_start=0, dof=None):
    path = _path()
    st = cp.initial_state(path)
    frames, _ = cp.sub_frames(path, t0, t1, 30.0, spp, 0.5, st, base)
    for i, f in enumerate(frames):
        f.spp_index = spp_start + i
        if dof is not None:  # keep the base frame's depth of field: the path's keyframes have none
            f.dof, f.focus_z = dof
    return frames


def _tonemap():
    return cp.default_tonemap(linear=True)


def _chain(r, frames, tm, acc, stream):
    """render_frame's sequence per sub-frame through the existing entry points: clear, nsb_render, nsb_accumulate; then nsb_tonemap."""
    import torch

    fb = torch.empty_like(acc)
    depth = torch.empty(acc.shape[:2], dtype=torch.float32, device=acc.device)
    out = torch.empty_like(acc)
    with torch.cuda.stream(stream):
        for f in frames:
            fb.zero_()
            depth.zero_()
            abi.check(r.lib, r.lib.nsb_render(r.ctx, C.byref(f), fb.data_ptr(), depth.data_ptr(), stream.cuda_stream), "nsb_render")
            abi.check(r.lib, r.lib.nsb_accumulate(r.ctx, fb.data_ptr(), acc.data_ptr(), f.width, f.height, f.spp_index, tm.color_space, stream.cuda_stream),
                      "nsb_accumulate")
        abi.check(r.lib, r.lib.nsb_tonemap(r.ctx, acc.data_ptr(), out.data_ptr(), frames[0].width, frames[0].height, C.byref(tm), stream.cuda_stream),
                  "nsb_tonemap")
    return out


def _same_bits(a, b):
    return np.array_equal(a.cpu().numpy().view(np.uint32), b.cpu().numpy().view(np.uint32))


@pytest.fixture(scope="module")
def maps():
    import torch

    env, dist = syn.make_envmap(), syn.make_distortion_map()
    return {"env_dev": torch.from_numpy(env).cuda(), "dist_dev": torch.from_numpy(dist).cuda()}


class _DevPtr:  # what CASES reads from a map (.ctypes.data, .shape), pointing at device memory
    def __init__(self, t):
        self.shape = tuple(t.shape)
        self.ctypes = type("p", (), {"data": t.data_ptr()})()


ACCUMULATE_CASES = {  # name: (frame case, spp, first spp_index, fp32 accumulators, edits, side stream)
    "plain_n8": ("plain", 8, 0, False, False, False),
    "plain_n1": ("plain", 1, 0, False, False, False),
    "plain_n33": ("plain", 33, 0, False, False, False),
    "fp32_n8": ("plain", 8, 0, True, False, False),
    "cage_membrane_n8": ("plain", 8, 0, False, True, False),
    "dof_n8": ("dof", 8, 0, False, False, False),
    "envmap_n8": ("envmap", 8, 0, False, False, False),
    "lens_n8": ("iterative", 8, 0, False, False, False),
    "continued_from_8": ("plain", 8, 8, False, False, False),
    "side_stream_n8": ("plain", 8, 0, False, False, True),
}


@pytest.mark.parametrize("name", list(ACCUMULATE_CASES))
def test_render_accumulate_equals_the_chain(scene, renderer, maps, name):
    import torch

    model, _ = scene
    case, spp, spp0, fp32, edits, side = ACCUMULATE_CASES[name]
    base = syn.make_frame(model, syn.orbit_cameras(120)[17], W, H, apply_operators=edits)
    dof = None
    if case != "plain":
        base = CASES[case](base, {"env": _DevPtr(maps["env_dev"]), "dist": _DevPtr(maps["dist_dev"])})
        dof = (base.dof, base.focus_z) if case == "dof" else None
    frames = _sub_frames(base, spp, spp_start=spp0, dof=dof)
    tm = _tonemap()
    stream = torch.cuda.Stream() if side else torch.cuda.current_stream()
    try:
        if fp32:
            renderer.set_mlp_accumulator(abi.NSB_MLP_ACC_F32)
        if edits:
            renderer.set_edit_operators([fx.make_cage(model, (0.5, 0.62, 0.78), (0.17, 0.17, 0.17), membrane_seed=5).to_op()])
        seed_acc = torch.rand((H, W, 4), device="cuda")  # what a continued accumulation starts from
        acc_a, acc_b = seed_acc.clone(), seed_acc.clone()
        stream.wait_stream(torch.cuda.current_stream())
        want = _chain(renderer, frames, tm, acc_a, stream)
        got_acc, got = renderer.render_accumulate(frames, tm, accumulate=acc_b, stream=stream.cuda_stream)
        stream.synchronize()
        assert _same_bits(got_acc, acc_a) and _same_bits(got, want)
        assert float(want[..., 3].mean()) > 0.05  # something was rendered
        if spp0 == 0:
            assert not _same_bits(acc_a, seed_acc)
    finally:
        renderer.set_mlp_accumulator(abi.NSB_MLP_ACC_F16)
        renderer.reset_edit_operators()


def test_no_allocation_after_the_first_call(scene, renderer):
    import torch

    model, _ = scene
    frames = _sub_frames(syn.make_frame(model, syn.orbit_cameras(120)[17], 320, 180), 4)
    tm = _tonemap()
    acc = torch.empty((180, 320, 4), device="cuda")
    out = torch.empty_like(acc)
    renderer.render_accumulate(frames, tm, accumulate=acc, out=out)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(10):
        renderer.render_accumulate(frames, tm, accumulate=acc, out=out)
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == free0
    small = _sub_frames(syn.make_frame(model, syn.orbit_cameras(120)[17], 64, 36), 2)  # a smaller size reuses the buffers
    renderer.render_accumulate(small, tm)
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == free0


def _bad_frames(model):
    def mk(**kw):
        f = syn.make_frame(model, syn.orbit_cameras(120)[17], W, H)
        for k, v in kw.items():
            setattr(f, k, v)
        return f

    return {
        "width": mk(width=0), "tiles": mk(tile_world=0), "mode": mk(render_mode=2), "distortion_mode": mk(camera_distortion_mode=3),
        "slice": mk(focus_z=-1.0), "dof": mk(dof=0.1, focus_z=0.0), "activation": mk(rgb_activation=9),
        "envmap": syn.set_maps(mk(), envmap_ptr=16, envmap_shape=(0, 4)),
    }


def test_argument_errors_match_nsb_render_and_enqueue_nothing(scene, renderer):
    import torch

    from nerfshop_b200.renderer import NerfRenderer

    model, _ = scene
    good = _sub_frames(syn.make_frame(model, syn.orbit_cameras(120)[17], W, H), 4)
    tm = _tonemap()
    acc = torch.full((H, W, 4), 7.0, device="cuda")
    out = torch.full((H, W, 4), 7.0, device="cuda")
    fb = torch.zeros_like(acc)
    depth = torch.zeros((H, W), device="cuda")
    lib, ctx = renderer.lib, renderer.ctx
    for name, bad in _bad_frames(model).items():
        want = lib.nsb_render(ctx, C.byref(bad), fb.data_ptr(), depth.data_ptr(), None)
        assert want != abi.NSB_OK, name
        arr = (abi.NsbFrame * 4)(good[0], good[1], bad, good[3])
        assert lib.nsb_render_accumulate(ctx, arr, 4, C.byref(tm), acc.data_ptr(), out.data_ptr(), None) == want, name
        assert b"sub-frame 2" in lib.nsb_last_error()
    other = syn.make_frame(model, syn.orbit_cameras(120)[17], W + 16, H)  # sizes differ
    arr = (abi.NsbFrame * 2)(good[0], other)
    assert lib.nsb_render_accumulate(ctx, arr, 2, C.byref(tm), acc.data_ptr(), out.data_ptr(), None) == abi.NSB_ERR_INVALID
    arr = (abi.NsbFrame * 4)(*good)
    bad_tm = _tonemap()
    bad_tm.tonemap_curve = 7
    assert lib.nsb_render_accumulate(ctx, arr, 4, C.byref(bad_tm), acc.data_ptr(), out.data_ptr(), None) == abi.NSB_ERR_INVALID
    assert lib.nsb_render_accumulate(ctx, arr, 0, C.byref(tm), acc.data_ptr(), out.data_ptr(), None) == abi.NSB_ERR_INVALID
    assert lib.nsb_render_accumulate(ctx, arr, 4, None, acc.data_ptr(), out.data_ptr(), None) == abi.NSB_ERR_INVALID
    assert lib.nsb_render_accumulate(ctx, arr, 4, C.byref(tm), None, out.data_ptr(), None) == abi.NSB_ERR_INVALID
    torch.cuda.synchronize()
    assert bool((acc == 7.0).all()) and bool((out == 7.0).all())
    empty = NerfRenderer(0)  # no model: NSB_ERR_STATE, as nsb_render
    try:
        assert empty.lib.nsb_render(empty.ctx, C.byref(good[0]), fb.data_ptr(), depth.data_ptr(), None) == abi.NSB_ERR_STATE
        assert empty.lib.nsb_render_accumulate(empty.ctx, arr, 4, C.byref(tm), acc.data_ptr(), out.data_ptr(), None) == abi.NSB_ERR_STATE
    finally:
        empty.close()
    for n_channels, ok in ((4, abi.NSB_OK), (3, abi.NSB_OK), (2, abi.NSB_ERR_INVALID), (1, abi.NSB_ERR_INVALID)):
        px = torch.empty(H * W * 4 + 4, dtype=torch.uint8, device="cuda")
        assert lib.nsb_frame_to_rgba8(ctx, out.data_ptr(), W, H, 0.0, n_channels, px.data_ptr(), None) == ok
    assert lib.nsb_frame_to_rgba8(ctx, out.data_ptr(), W, H, 0.0, 4, px.data_ptr() + 1, None) == abi.NSB_ERR_INVALID  # uchar4 alignment
    assert lib.nsb_frame_to_rgba8(ctx, out.data_ptr(), 0, H, 0.0, 4, px.data_ptr(), None) == abi.NSB_ERR_INVALID
    torch.cuda.synchronize()


# ---- nsb_frame_to_rgba8 against run.py + write_image (scripts/common.py:122-178), transcribed -------------------------------------------
def _write_image_bytes(frame, exposure, pow_nudge=0):
    """np.clip(frame * 2**exposure, 0, 1) then write_image's 8-bit pixels, as numpy computes them on float32 arrays. pow_nudge = +-1
    moves the x**(1/2.4) result by one ulp (the device's powf is not the host's). NaN gives 0 (numpy's cast of NaN is undefined)."""
    with np.errstate(all="ignore"):
        img = np.clip(np.asarray(frame, np.float32) * 2 ** exposure, 0.0, 1.0)
        img = np.copy(img)
        img[..., 0:3] = np.divide(img[..., 0:3], img[..., 3:4], out=np.zeros_like(img[..., 0:3]), where=img[..., 3:4] != 0)
        x = img[..., 0:3]
        p = x ** (1.0 / 2.4)
        if pow_nudge:
            p = np.nextafter(p, np.float32(np.inf if pow_nudge > 0 else -np.inf))
        img[..., 0:3] = np.where(x > 0.0031308, 1.055 * p - 0.055, 12.92 * x)
        q = np.clip(img, 0.0, 1.0) * 255.0 + 0.5
        return np.where(np.isnan(q), 0, q).astype(np.uint8)


def _crafted():
    lim = np.float32(0.0031308)
    vals = np.concatenate([
        np.array([0.0, -0.0, -1.0, -1e-30, 1e-30, 1.0, 1.5, 1e30, np.inf, -np.inf, np.nan, 0.5, 0.999, 1.0 - 2 ** -24], np.float32),
        np.nextafter(np.full(8, lim), np.float32(0)), np.full(1, lim), np.nextafter(np.full(8, lim), np.float32(1)),
        np.linspace(0.0, 1.0, 4097, dtype=np.float32), np.random.default_rng(3).uniform(-0.5, 1.5, 20000).astype(np.float32),
    ])
    alphas = np.array([0.0, 1e-38, 1e-30, 1e-7, 0.01, 0.5, 1.0, 1.2, -0.3, np.nan], np.float32)
    rng = np.random.default_rng(4)
    n = vals.size
    out = np.zeros((n, 4), np.float32)
    out[:, 0] = vals
    out[:, 1] = rng.permutation(vals)
    out[:, 2] = vals[::-1]
    out[:, 3] = np.concatenate([alphas[np.arange(n) % alphas.size][: n // 2], rng.uniform(0, 1, n - n // 2).astype(np.float32)])
    out[:, :3] *= np.where(np.isfinite(out[:, 3:4]) & (out[:, 3:4] > 0), out[:, 3:4], 1.0)  # premultiplied where that means something
    w = 128
    rows = (n + w - 1) // w
    pad = np.zeros((rows * w - n, 4), np.float32)
    return np.concatenate([out, pad]).reshape(rows, w, 4)


def _check_bytes(got, frame, exposure, n_channels=4):
    want = _write_image_bytes(frame, exposure)[..., :n_channels]
    lo = _write_image_bytes(frame, exposure, -1)[..., :n_channels]
    hi = _write_image_bytes(frame, exposure, +1)[..., :n_channels]
    diff = got != want
    boundary = diff & ((got == lo) | (got == hi))
    print(f"rgba8: {int(diff.sum())} of {diff.size} bytes differ from numpy, all within one powf ulp of a quantisation boundary: "
          f"{int(boundary.sum())}")
    assert np.array_equal(diff, boundary)
    assert diff.sum() <= max(4, diff.size // 10000)


@pytest.mark.parametrize("exposure", [0.0, 1.0, -0.5])
def test_frame_to_rgba8_matches_write_image_on_crafted_input(renderer, exposure):
    import torch

    frame = _crafted()
    dev = torch.from_numpy(frame).cuda()
    for n_channels in (4, 3):
        got = renderer.frame_to_rgba8(dev, exposure, n_channels).cpu().numpy()
        assert got.shape == frame.shape[:2] + (n_channels,)
        _check_bytes(got, frame, exposure, n_channels)


def test_frame_to_rgba8_matches_write_image_on_rendered_frames(scene, renderer):
    model, _ = scene
    base = syn.make_frame(model, syn.orbit_cameras(120)[17], W, H)
    frames = _sub_frames(base, 8)
    for tm in (cp.default_tonemap(linear=True), cp.default_tonemap(linear=False)):
        tm.background_color[:] = [0.1, 0.2, 0.3, 0.0]  # transparent background: partial alpha survives
        _, out = renderer.render_accumulate(frames, tm)
        a = out[..., 3].cpu().numpy()
        assert ((a > 0.05) & (a < 0.95)).any()
        for exposure in (0.0, 0.75):
            _check_bytes(renderer.frame_to_rgba8(out, exposure).cpu().numpy(), out.cpu().numpy(), exposure)


# ---- render_video --------------------------------------------------------------------------------------------------------------------
def test_render_video(scene, renderer, tmp_path):
    import torch

    model, _ = scene
    path = _path()
    base = syn.make_frame(model, syn.orbit_cameras(120)[17], 320, 180)
    probe = syn.make_frame(model, syn.orbit_cameras(120)[30], 160, 90)
    before = renderer.render(probe)[0].clone()
    runs = []
    for run in range(2):
        out_dir = str(tmp_path / f"run{run}")
        names = cp.render_video(renderer, base, path, n_seconds=1, fps=6, spp=4, out_dir=out_dir, smoothing=True, exposure=0.25)
        assert [os.path.basename(n) for n in names] == ["%04d.png" % i for i in range(6)]
        runs.append([open(n, "rb").read() for n in names])
    assert runs[0] == runs[1]
    # every file holds the device's bytes for the frame sub_frames describes, in run.py's order of calls
    st = cp.initial_state(path)
    tm = cp.default_tonemap(linear=True)
    for i in range(6):
        st.camera_smoothing = i > 0
        frames, _ = cp.sub_frames(path, i / 6, (i + 1) / 6, 6, 4, 0.5, st, base)
        if i == 0:  # frame 0: the shutter runs from the path's start to t = 1/6, the focal length and focus come from the mid times
            assert len(frames) == 4 and [f.spp_index for f in frames] == [0, 1, 2, 3]
            assert np.array_equal(np.array(frames[0].camera0, np.float32), np.array(cp.frame_from_keyframe(base, path.eval_camera_path(0.0)).camera0, np.float32))
        _, rgba = renderer.render_accumulate(frames, tm)
        px = renderer.frame_to_rgba8(rgba, 0.25).cpu().numpy()
        assert np.array_equal(decode_png(runs[0][i]), px), i
    assert runs[0][0] != runs[0][5]
    torch.cuda.synchronize()
    after = renderer.render(probe)[0]
    assert _same_bits(before, after)


# ---- against the reference's own CUDA path ------------------------------------------------------------------------------------------
def _ref_video_available():
    from oracle import ref_video_build

    return ref_video_build.build() is not None


# tonemaps other than render_frame's default: (curve, input colour space, output colour space, clamp, exposure)
_TONEMAPS = {
    "reinhard_srgb_clamp": (abi.NSB_TONEMAP_REINHARD, abi.NSB_COLOR_LINEAR, abi.NSB_COLOR_SRGB, 1, 0.0),
    "aces_exposure": (abi.NSB_TONEMAP_ACES, abi.NSB_COLOR_LINEAR, abi.NSB_COLOR_LINEAR, 0, 1.3),
    "hable_srgb_accumulate": (abi.NSB_TONEMAP_HABLE, abi.NSB_COLOR_SRGB, abi.NSB_COLOR_SRGB, 0, 0.0),
    "visposneg": (abi.NSB_TONEMAP_IDENTITY, abi.NSB_COLOR_VISPOSNEG, abi.NSB_COLOR_LINEAR, 0, -0.5),
}


@pytest.mark.skipif(not (_ref_video_available() or os.path.isdir(os.path.join(os.path.dirname(__file__), "golden", "ref", "test_gpu_camera_path"))),
                    reason="neither oracle/_ref nor stored reference results (tests/golden/ref/)")
@pytest.mark.parametrize("edits, tonemap", [(False, None), (True, None)] + [(False, k) for k in _TONEMAPS] + [(True, "reinhard_srgb_clamp")],
                         ids=["plain", "e1"] + [f"plain_{k}" for k in _TONEMAPS] + ["e1_reinhard_srgb_clamp"])
def test_render_accumulate_vs_reference_cuda(scene, renderer, edits, tonemap):
    """The same sub-frame cameras through the reference's clear_frame -> render_nerf -> accumulate_kernel -> tonemap_kernel, once per
    sub-frame as render_frame runs them (oracle/ref_video_driver_cuda.cu): L-inf 0 without edits (as the frame-domain tests), <= 1e-3 with
    E1 (DESIGN §6), under render_frame's default tonemap and under every curve, sRGB accumulation and output, clamping, exposure and
    VisPosNeg. Where oracle/_ref is absent the stored results of the reference are replayed."""
    import ref_golden

    from oracle import ref_video

    model, occ = scene
    base = syn.make_frame(model, syn.orbit_cameras(120)[17], W, H, apply_operators=edits)
    frames = _sub_frames(base, 8)
    tm = _tonemap()
    tm.background_color[:] = [0.1, 0.2, 0.3, 0.5]
    digest = []
    if tonemap is not None:
        tm.tonemap_curve, tm.color_space, tm.output_color_space, tm.clamp_output_color, tm.exposure = _TONEMAPS[tonemap]
        digest = [np.array(_TONEMAPS[tonemap], np.float32)]
    ops = [op.to_op() for op in fx.e1(model)] if edits else None
    cams = np.array([[list(f.camera0), list(f.camera1), list(f.focal_length) + [0.0] * 10] for f in frames], np.float32)  # the inputs' digest
    try:
        renderer.set_edit_operators(ops or [])
        want = ref_golden._call(_ref_video_available(), lambda c, *_: ref_video.render_to_cpu(occ, ops, frames, renderer, tm), cams, *digest)
        _, got = renderer.render_accumulate(frames, tm)
        got = got.cpu().numpy()
    finally:
        renderer.reset_edit_operators()
    got, want = ref_golden.ref.match(got, want)
    err = float(np.abs(got - want).max())
    print(f"\nrender_accumulate vs the reference's render_frame sequence ({'E1' if edits else 'plain'}, {tonemap or 'default tonemap'}, 8 sub-frames): "
          f"L-inf {err:.3e}")
    assert float(want[..., 3].mean()) > 0.05
    assert err <= (1e-3 if edits else 0.0)
