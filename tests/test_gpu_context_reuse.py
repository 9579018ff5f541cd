"""A context that has been used before computes what a fresh one computes: a re-uploaded model, framebuffers and ray buffers that
had to grow, membrane scratch sized for another cage, and contexts created and destroyed in a row. Each case makes its own contexts."""
import numpy as np
import pytest

import edit_fixtures as fx
from nerfshop_b200 import abi
from nerfshop_b200 import synthetic as syn

pytestmark = pytest.mark.gpu


@pytest.fixture
def make_renderer(scene, built_lib):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nerfshop_b200.renderer import NerfRenderer

    made = []

    def make(with_scene=True):
        r = NerfRenderer(0)
        made.append(r)
        if with_scene:
            model, occ = scene
            r.upload_model(model.desc, model.params)
            r.upload_occupancy(occ)
        return r

    yield make
    for r in made:
        r.close()


def _fresh_host_frame(make_renderer, f):
    r = make_renderer()
    fb, depth = r.render_to_cpu(f)
    r.close()
    return fb, depth


def test_model_reupload_matches_a_fresh_context(scene, make_renderer):
    model, _ = scene
    other = syn.make_model(seed=7)
    f = syn.make_frame(model, syn.orbit_cameras(120)[17], 320, 180)
    want = _fresh_host_frame(make_renderer, f)
    r = make_renderer()
    r.upload_model(other.desc, other.params)
    mid, _ = r.render_to_cpu(f)
    assert not np.array_equal(mid, want[0])  # the other model is the one rendered
    r.upload_model(model.desc, model.params)
    fb, depth = r.render_to_cpu(f)
    assert np.array_equal(fb, want[0]) and np.array_equal(depth, want[1])


def test_grown_buffers_match_a_fresh_context(scene, make_renderer):
    """Small, 1080p, general-camera, small again: the ray list, the general-camera ray buffer and both host-delivery framebuffer sets
    grow on the way, and every frame equals the one a fresh context renders."""
    import torch

    model, _ = scene
    cams = syn.orbit_cameras(120)
    general = syn.set_camera_distortion(syn.make_frame(model, cams[40], 960, 540), abi.NSB_CAMERA_DISTORTION_ITERATIVE, [0.08, -0.02, 0.003, -0.002])
    frames = [syn.make_frame(model, cams[5], 320, 180), syn.make_frame(model, cams[17], 1920, 1080), general, syn.make_frame(model, cams[90], 320, 180)]
    want = [_fresh_host_frame(make_renderer, f) for f in frames]
    r = make_renderer()
    for f, (fb_w, depth_w) in zip(frames, want):
        fb, depth = r.render_to_cpu(f)
        assert np.array_equal(fb, fb_w) and np.array_equal(depth, depth_w)
    host = [(torch.zeros((f.height, f.width, 4)).pin_memory(), torch.zeros((f.height, f.width)).pin_memory()) for f in frames]
    tickets = [r.render_to_cpu_async(f, *h) for f, h in zip(frames, host)]  # the framebuffers grow while earlier copies are in flight
    for t in tickets:
        r.wait_host_frame(t)
    for (fb, depth), (fb_w, depth_w) in zip(host, want):
        assert np.array_equal(fb.numpy(), fb_w) and np.array_equal(depth.numpy(), depth_w)


def test_membrane_scratch_resized_matches_a_fresh_context(scene, make_renderer):
    model, _ = scene
    op = fx.e1(model)[0]
    rng = np.random.default_rng(3)
    nv, nc = op.mvc.shape

    def inputs(k):  # the blend of the first k cage vertices
        d_in, d_out = rng.uniform(0.5, 40.0, (2, nc)).astype(np.float32)
        s_in, s_out = rng.uniform(-0.5, 0.5, (2, nc, 27)).astype(np.float32)
        return np.ascontiguousarray(op.mvc[:, :k]), d_in[:k], d_out[:k], s_in[:k], s_out[:k]

    def fresh(args):
        r = make_renderer(with_scene=False)
        r.set_edit_operators([op.to_op()])
        out = r.cage_set_membrane(0, *args)
        r.close()
        return out

    all_cv, fewer_cv = inputs(nc), inputs(nc - 3)
    want_all, want_fewer = fresh(all_cv), fresh(fewer_cv)
    assert not np.array_equal(want_all[0], want_fewer[0])
    r = make_renderer(with_scene=False)
    r.set_edit_operators([op.to_op()])
    for args, want in ((all_cv, want_all), (fewer_cv, want_fewer), (all_cv, want_all)):
        got = r.cage_set_membrane(0, *args)
        assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(got, want))


def test_create_render_destroy_in_a_row(scene, make_renderer):
    model, _ = scene
    f = syn.make_frame(model, syn.orbit_cameras(120)[17], 128, 72)
    first = None
    for _ in range(10):
        r = make_renderer()
        fb, depth = r.render_to_cpu(f)
        assert r.stats().n_samples > 0
        r.close()
        if first is None:
            first = (fb, depth)
        assert np.array_equal(fb, first[0]) and np.array_equal(depth, first[1])
