"""The CUDA path over the frame parameter space of tests/frame_domain.py: ray-box entry from outside the render AABB, crop boxes, rolling
shutter, lens fields, jitter indices, the march's cone and train AABB, transmittance, activations, linear colours and every render mode.

  * nsb_march_trace against the CPU oracle: bit for bit (t, dt, position, mip, cell), every case, every pixel;
  * nsb_render against the oracle: the frame tolerance of test_gpu_parity.py (relative where a debug colour exceeds 1), the same ray and
    live-ray counts, and the case's minimum share of hit pixels;
  * the sample stream against the reference's own CUDA kernels (oracle/_ref/libnerfshop_ref_cuda.so): counts, t after `t += dt`, warped
    position and warped dt bit for bit, once per distinct march (frame_domain.MARCH_CASES);
  * the frame against the reference's render_nerf: RGBA and depth bit for bit under the default fp16-accumulator policy, and again under
    fp32 accumulators for the activation, transmittance and linear-colour cases.
Where oracle/_ref is absent the reference's stored results (tests/golden/ref/) are replayed.
"""
import numpy as np
import pytest

import frame_domain as fd
from nerfshop_b200 import abi
from ref_golden import ref
from test_gpu_march_edge_inputs import _march_bit_exact
from test_gpu_parity import _compare_frames

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not ref.cuda_usable("test_gpu_frame_domain"), reason="neither oracle/_ref nor stored reference results (tests/golden/ref/)")

MS = 32
POLICIES = {"f16": abi.NSB_MLP_ACC_F16, "f32": abi.NSB_MLP_ACC_F32}
FRAME_RUNS = [(n, "f16") for n in fd.CASES] + [(n, "f32") for n in fd.FP32_CASES]


@pytest.fixture(scope="module")
def ref_cuda(scene):
    rc = ref.RefCuda(scene[1])
    yield rc
    rc.close()


@pytest.mark.parametrize("name", list(fd.CASES))
def test_march_bit_exact_vs_oracle(scene, oracle, renderer, name):
    f = fd.frame(scene[0], name)
    _, _, cnt = _march_bit_exact(oracle, renderer, f)
    assert (cnt > 0).mean() >= fd.MIN_HIT[name]  # a hit pixel has at least one sample


@pytest.mark.parametrize("name", list(fd.CASES))
def test_frame_vs_oracle(scene, oracle, renderer, name):
    """The depth is that of a ray's max-weight sample. Under a logistic density (act_exp_logistic) sigma stays below 1, so neighbouring
    samples carry nearly equal weights and the network's rounding (1e-4) picks the maximum among them: there the depth is held to the
    share of hit pixels whose maximum moved, and the RGBA to the frame tolerance as everywhere."""
    f = fd.frame(scene[0], name)
    fb_o, depth_o, st_o, margin = oracle.render(f, want_margin=True)
    fb, depth = renderer.render(f)
    st = renderer.stats()
    fb, depth = fb.cpu().numpy(), depth.cpu().numpy()
    s = np.maximum(1.0, np.abs(fb_o))  # depth, distance and cost colours exceed 1: the 1e-3 tolerance is relative there
    if f.density_activation == abi.NSB_ACT_LOGISTIC:
        _compare_frames(fb / s, depth_o, fb_o / s, depth_o, margin)
        assert ((depth_o < 1e9) == (depth < 1e9)).mean() > 0.9995
        hit = (depth_o < 1e9) & (depth < 1e9)
        moved = np.abs(depth - depth_o)[hit] > 1e-3 * np.abs(depth_o[hit]).max() + 1e-4
        print(f"\n{name}: max-weight sample moved on {moved.sum()} of {hit.sum()} hit pixels, by up to {np.abs(depth - depth_o)[hit].max():.4f}")
        assert moved.mean() <= 0.02
    else:
        _compare_frames(fb / s, depth, fb_o / s, depth_o, margin)
    assert (st.n_rays, st.n_rays_alive) == (st_o.n_rays, st_o.n_rays_alive)
    assert (fb[..., 3] != 0).mean() >= fd.MIN_HIT[name]


@needs_ref
@pytest.mark.parametrize("name", fd.MARCH_CASES)
def test_sample_stream_bit_exact_vs_reference_kernels(scene, renderer, ref_cuda, name):
    f = fd.frame(scene[0], name)
    pix = fd.pixels(f, 250)
    rec, _, cnt = renderer.march_trace(f, pix, MS)
    rec_r, _, cnt_r = ref_cuda.march_trace(f, pix, MS)
    frac = ref.fraction(cnt_r)  # a stored reference result keeps a seeded sample of the rays: compare on those
    rec, rec_r = ref.match(rec, rec_r)
    cnt, cnt_r = ref.match(cnt, cnt_r)
    assert np.array_equal(np.minimum(cnt, MS), cnt_r)
    valid = np.arange(MS)[None, :] < cnt_r[:, None]
    assert valid.sum() > 1000 * frac
    t_after = (rec[..., 0] + rec[..., 1]).astype(np.float32)  # payload.t after `t += dt` (generate_next_nerf_network_inputs)
    np.testing.assert_array_equal(t_after[valid], rec_r[..., 7][valid])
    amin, amax = np.array(list(f.train_aabb_min), np.float32), np.array(list(f.train_aabb_max), np.float32)
    wp = ((rec[..., 2:5] - amin) / (amax - amin)).astype(np.float32)  # warp_position: one sub, one div per component
    np.testing.assert_array_equal(wp[valid], rec_r[..., 0:3][valid])
    min_step = np.float32(np.float32(1.73205080757) / np.float32(1024.0))
    wdt = ((rec[..., 1] - min_step) / (min_step * np.float32(16.0) - min_step)).astype(np.float32)  # warp_dt
    np.testing.assert_array_equal(wdt[valid], rec_r[..., 3][valid])


@needs_ref
@pytest.mark.parametrize("name,policy", FRAME_RUNS)
def test_frame_identical_to_reference_render_nerf(scene, renderer, ref_cuda, name, policy):
    import torch

    f = fd.frame(scene[0], name)
    try:
        renderer.set_mlp_accumulator(POLICIES[policy])
        fb, depth = renderer.render(f)
        fb_r, depth_r, _ = ref_cuda.render(f, renderer)
        torch.cuda.synchronize()
    finally:
        renderer.set_mlp_accumulator(abi.NSB_MLP_ACC_F16)
    assert (fb[..., 3] != 0).float().mean().item() >= fd.MIN_HIT[name]
    fb, fb_r = ref.match(fb, fb_r)  # a stored reference frame keeps a seeded sample of its rows
    depth, depth_r = ref.match(depth, depth_r)
    diff = (fb - fb_r).abs().amax(-1)
    assert torch.equal(fb, fb_r), f"{name} {policy}: {int((diff > 0).sum())} pixels differ, L-inf {diff.max().item():.3e}"
    assert torch.equal(depth, depth_r), f"{name} {policy}: depth differs on {int((depth != depth_r).sum())} pixels"
