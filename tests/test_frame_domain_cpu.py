"""The CPU oracle against the reference's own sources compiled for the CPU, over the frame parameter space of tests/frame_domain.py.

The march runs once per distinct march (frame_domain.MARCH_CASES: a case that differs from an earlier one only in composite or shading
fields marches the same samples), the frame once per case. The rules are those of test_oracle_vs_ref.py: the same rays enter and each
takes the same number of occupied samples; the t stream is identical; warped positions agree to a few ulps (the camera matrix product and the normalisation are contracted into FMAs as each
compiler chooses). Where the camera is outside the render AABB the first t is box_ray_tmin's, computed on a direction whose bits that
contraction already moves: there a ray's t stream may start up to 8 ulps away, and the count of such rays is printed. Frames: the same
hit set, and <= 1e-3 away from pixels whose accumulated alpha lies within float noise of the termination threshold.
Where the reference's sources are absent, its stored results (tests/golden/ref/) are replayed.
"""
import numpy as np
import pytest

import frame_domain as fd
from nerfshop_b200 import abi
from ref_golden import ref

pytestmark = pytest.mark.skipif(not ref.usable("test_frame_domain_cpu"), reason="neither oracle/_ref nor stored reference results (tests/golden/ref/)")

MS = 32


def ulps(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64))


@pytest.mark.parametrize("name", fd.MARCH_CASES)
def test_march_vs_reference_kernels(scene, oracle, name):
    model, occ = scene
    f = fd.frame(model, name)
    pix = fd.pixels(f, 250)
    rec_o, _, cnt_o = oracle.march_trace(f, pix, MS)
    rec_r, _, cnt_r, _ = ref.march_trace(f, occ, pix, MS)
    frac = ref.fraction(cnt_r)
    rec_o, rec_r = ref.match(rec_o, rec_r)
    cnt_o, cnt_r = ref.match(cnt_o, cnt_r)
    assert np.array_equal(np.minimum(cnt_o, MS), cnt_r)
    valid = np.arange(MS)[None, :] < cnt_r[:, None]
    assert valid.sum() > 1000 * frac, valid.sum()
    t_after = (rec_o[..., 0] + rec_o[..., 1]).astype(np.float32)  # payload.t after `t += dt`
    dt_ulps = np.where(valid, ulps(t_after, rec_r[..., 7]), 0)
    moved = dt_ulps.max(axis=1) > 0
    amin, amax = np.array(list(f.train_aabb_min), np.float32), np.array(list(f.train_aabb_max), np.float32)
    dpos = np.abs(((rec_o[..., 2:5] - amin) / (amax - amin)).astype(np.float32) - rec_r[..., 0:3])[valid] / 2.0 ** -24
    outside = fd.camera_outside_render_box(f)
    print(f"\n{name}: {valid.sum()} samples on {(cnt_r > 0).sum()} rays; camera outside the render AABB: {outside}; rays whose t stream "
          f"differs {moved.sum()} (entry max {dt_ulps[:, 0].max()} ulp, stream max {dt_ulps.max()} ulp); warped positions max {dpos.max():.1f} ulp of 1.0")
    if outside:
        assert dt_ulps[:, 0].max() <= 8 and dt_ulps.max() <= 8
        assert (dt_ulps[moved, 0] > 0).all()  # a ray whose entry agrees keeps the same stream
    else:
        assert not moved.any()
    assert dpos.max() <= 8


@pytest.mark.parametrize("name", list(fd.CASES))
def test_frame_vs_reference_render_nerf(scene, oracle, name):
    model, occ = scene
    f = fd.frame(model, name)
    fb_o, d_o, st, margin = oracle.render(f, want_margin=True)
    fb_r, d_r, info = ref.render(f, occ, lambda c: oracle.inference(c))
    assert (fb_o[..., 3] != 0).mean() >= fd.MIN_HIT[name]
    # the debug colours (depth, distance, cost) are not in [0, 1]: the 1e-3 contract is applied relative to the value there
    err = (np.abs(fb_o - fb_r) / np.maximum(1.0, np.abs(fb_o))).max(-1)
    ok = (margin > 2e-5) | (fb_o[..., 3] == 0)
    print(f"\n{name}: L-inf {err[ok].max():.3e} ({(~ok).sum()} threshold pixels apart, worst of them {err[~ok].max() if (~ok).any() else 0:.3e}); "
          f"pixels > 1e-4: {(err > 1e-4).sum()} of {err.size}")
    assert (err[~ok] > 1e-3).sum() <= 2  # a threshold pixel may take the other branch; measured: none does
    assert np.array_equal(fb_o[..., 3] != 0, fb_r[..., 3] != 0)  # same hit set (compact_kernel_nerf's filter)
    if f.render_mode == abi.NSB_RENDER_SHADE:
        assert err[ok].max() <= 1e-3
    else:  # a position an ulp apart can move one sample across an occupancy cell face: the debug colours show it
        assert (err[ok] > 1e-3).sum() <= 2
    assert info["n_calls"] % 2 == 0 and info["n_inferred"] >= 2 * st.n_samples
