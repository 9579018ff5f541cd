"""Occupancy-march inputs the orbit cameras never produce, CUDA path against the CPU oracle (DESIGN.md §3):
  * rays with a zero direction component (reciprocal direction ±inf), from cameras looking down the axes
  * a camera at the AABB centre (positions a hair from the centre: the smallest mip_from_pos arguments a ray reaches)
  * a camera inside the fox AABB at negative coordinates, whose rays cross every cascade boundary
  * a train AABB whose extent is not a power of two (warp_position divides instead of multiplying by 2^-k; the frame is compared
    with the oracle's within the frame tolerance)
The march is compared bit for bit: t, dt, position, mip and cell index."""
import numpy as np
import pytest

from nerfshop_b200 import synthetic as syn

pytestmark = pytest.mark.gpu


def _march_bit_exact(oracle, renderer, f, max_samples=256, step=1):
    pix = np.arange(0, f.width * f.height, step, dtype=np.uint32)
    rec_o, idx_o, cnt_o = oracle.march_trace(f, pix, max_samples)
    rec_g, idx_g, cnt_g = renderer.march_trace(f, pix, max_samples)
    assert (cnt_o == cnt_g).all(), f"sample counts differ on {(cnt_o != cnt_g).sum()} rays"
    assert (idx_o == idx_g).all(), "mip / cell differ"
    assert (rec_o.view(np.uint32) == rec_g.view(np.uint32)).all(), "t/dt/pos bits differ"
    return rec_o, idx_o, cnt_o


@pytest.mark.parametrize("pos", [(0.5, 0.5, 2.3), (0.5, 0.5, -1.3), (2.3, 0.5, 0.5), (0.5, -1.3, 0.5)])
def test_march_axis_aligned_rays(scene, oracle, renderer, pos):
    """Odd resolution: the centre row and column of pixels have a direction component of exactly ±0."""
    model, _ = scene
    up = (0.0, 0.0, 1.0) if pos[0] == 0.5 and pos[2] == 0.5 else (0.0, 1.0, 0.0)
    f = syn.make_frame(model, syn.look_at(pos, up=up), 97, 55)
    rec, idx, cnt = _march_bit_exact(oracle, renderer, f)
    assert cnt.sum() > 1000


def test_march_camera_at_aabb_centre(scene, oracle, renderer):
    model, _ = scene
    f = syn.make_frame(model, syn.look_at((0.5, 0.5, 0.5), target=(0.5, 0.5, 1.5)), 97, 55)
    _, idx, cnt = _march_bit_exact(oracle, renderer, f)
    assert cnt.sum() > 1000
    first = idx[:, 0, 0][cnt > 0]
    assert (first == 0).any()  # samples near the centre sit in the finest cascade


def test_march_crosses_cascades_from_negative_coordinates(scene, oracle, renderer):
    model, _ = scene
    assert model.aabb_min.min() < -1.0  # fox scale: the AABB reaches negative coordinates
    f = syn.make_frame(model, syn.look_at((-1.2, -1.1, -1.3)), 96, 54)
    _, idx, cnt = _march_bit_exact(oracle, renderer, f, max_samples=1024)
    mips = {int(m) for r, c in zip(idx, cnt) for m in r[:c, 0]}
    assert len(mips) >= 2, f"cascades visited: {sorted(mips)}"


def test_render_train_aabb_extent_not_power_of_two(scene, oracle, renderer):
    """Extents 5 x 4 x 5 around the render AABB: only the y axis is a power of two, so the frame takes the dividing warp_position."""
    model, _ = scene
    f = syn.make_frame(model, syn.orbit_cameras(120)[40], 96, 54)
    f.train_aabb_min[0], f.train_aabb_max[0] = -1.5, 3.5
    f.train_aabb_min[2], f.train_aabb_max[2] = -2.0, 3.0
    fb_o, depth_o, st_o, margin = oracle.render(f, want_margin=True)
    fb, depth = renderer.render(f)
    fb, depth = fb.cpu().numpy(), depth.cpu().numpy()
    st = renderer.stats()
    assert st.n_rays_alive == st_o.n_rays_alive
    diff = np.abs(fb - fb_o).max(axis=-1)
    ambiguous = margin <= 2e-5  # the early-termination branch within float noise (tests/test_gpu_parity.py)
    assert (diff[~ambiguous] <= 1e-3).all(), f"L-inf RGBA {diff[~ambiguous].max():.2e}"
    assert ((diff > 1e-3) & ambiguous).sum() <= 2
