"""Frames over the NsbFrame parameter space: the case table of test_frame_domain_cpu.py and test_gpu_frame_domain.py.

CASES[name](f) edits a syn.make_frame(model, BASE_CAMERA, W, H) frame; `frame(model, name)` builds it. Each line says which code path of
ray generation (make_ray, box_ray_tmin), the march or the composite the case reaches. Every case renders something: MIN_HIT holds the
share of pixels each must hit (measured with the CPU oracle, about half of it is asserted), and a case that renders nothing fails.
"""
import types

import numpy as np

from nerfshop_b200 import abi
from nerfshop_b200 import synthetic as syn

W, H = 96, 54          # 54 rows: not a multiple of the 8-row tile
W_ODD, H_ODD = 97, 55  # odd: the centre row and column of pixels have a direction component of exactly +-0
BASE_CAMERA = syn.orbit_cameras(120)[17]
ORBIT = syn.orbit_cameras(120)
FOX_MIN, FOX_MAX = (-1.5, -1.5, -1.5), (2.5, 2.5, 2.5)
CROP_MIN, CROP_MAX = (-0.25, -0.1, -0.25), (1.25, 1.15, 1.25)  # render AABB strictly inside the train AABB, around the fox and the ground


def _camera(f, cam0, cam1=None):
    for name, cam in (("camera0", cam0), ("camera1", cam0 if cam1 is None else cam1)):
        flat = np.asarray(cam, np.float32).reshape(3, 4).T.reshape(-1)  # column-major, as make_frame
        getattr(f, name)[:] = [float(v) for v in flat]


def _size(f, w, h):
    f.width, f.height = w, h
    f.focal_length[0] = f.focal_length[1] = float(h)


def _render_aabb(f, mn, mx):
    f.render_aabb_min[:], f.render_aabb_max[:] = mn, mx


def _set(**kw):
    def edit(f):
        for k, v in kw.items():
            if isinstance(v, tuple):
                getattr(f, k)[:] = v
            else:
                setattr(f, k, v)
    return edit


def _all(*edits):
    def edit(f):
        for e in edits:
            e(f)
    return edit


def _cam(pos, target=(0.5, 0.5, 0.5), up=(0.0, 1.0, 0.0)):
    return lambda f: _camera(f, syn.look_at(pos, target, up))


def _outside_radius(r, a):
    return (0.5 + r * np.cos(a), 0.85, 0.5 + r * np.sin(a))


_ROLLING = lambda f: _camera(f, ORBIT[20], ORBIT[17])  # noqa: E731
_CROP = lambda f: _render_aabb(f, CROP_MIN, CROP_MAX)  # noqa: E731

CASES = {
    # ray-box entry: the first t comes from box_ray_tmin, not from the near distance
    "outside_box": _cam(_outside_radius(3.6, 0.7), target=(0.5, 0.85, 0.5)),                      # first t from box_ray_tmin
    "crop_outside": _CROP,                                                                        # enters and leaves the crop box mid-scene; IN_RANGE instantiation
    "crop_inside": _all(_CROP, _cam((1.0, 0.9, 1.1))),                                            # starts inside the crop box, exits through a crop face
    "axis_outside": _all(lambda f: _size(f, W_ODD, H_ODD), _cam((0.5, 0.5, 4.0))),                 # +-0 direction components (idir +-inf) with box entry
    "face_plane": _all(lambda f: _size(f, W_ODD, H_ODD), _cam((-1.5, 0.5, -3.0), target=(-1.5, 0.5, 0.5))),  # origin on the x = -1.5 face: 0/0 = NaN in the slab test
    # rolling shutter: ray_time's FMA chain and the camera0 / camera1 blend
    "rolling_shutter": _all(_ROLLING, _set(rolling_shutter=(0.1, 0.3, 0.2, 0.25), spp_index=3)),  # every term of ray_time, jittered
    "rolling_no_jitter": _all(_ROLLING, _set(rolling_shutter=(0.25, 0.5, -0.5, 0.0))),             # the rs[3] == 0 branch, ray_time outside [0, 1]
    "rolling_cam0": _all(_ROLLING, _set(rolling_shutter=(1.0, 0.0, 0.0, 0.0))),                    # the blend gives camera0 exactly
    # lens and sampling
    "lens": _set(screen_center=(0.37, 0.61), focal_length=(41.0, 77.0)),                           # off-centre, anisotropic, wide field of view
    "narrow": _set(focal_length=(8.0 * H, 8.0 * H)),                                              # near-parallel rays
    "snap": _set(snap_to_pixel_centers=1, spp_index=7),                                           # pixel offset of spp 0, jitter of spp 7
    "large_spp": _set(spp_index=(1 << 20) + 3),                                                   # ld_random_val's high index bits
    # march
    "cone_0": _set(cone_angle_constant=0.0),                                                      # constant step
    "cone_1_128": _set(cone_angle_constant=1.0 / 128.0),                                          # coarser cascades (1/64 reaches cascade 4: empty)
    "train_not_pow2": _set(train_aabb_min=(-1.5, -1.5, -2.0), train_aabb_max=(3.5, 2.5, 3.0)),    # extents 5 x 4 x 5: tinv_exact = 0, dividing warp_position
    # composite
    "min_T_0": _set(min_transmittance=0.0),                                                       # no early termination
    "min_T_0.3": _set(min_transmittance=0.3),                                                     # early termination
    "min_T_0.999": _set(min_transmittance=0.999),                                                 # terminates at the first weighty sample
    "act_none_relu": _set(rgb_activation=abi.NSB_ACT_NONE, density_activation=abi.NSB_ACT_RELU),              # raw rgb, ReLU density
    "act_exp_logistic": _set(rgb_activation=abi.NSB_ACT_EXPONENTIAL, density_activation=abi.NSB_ACT_LOGISTIC),  # clamped exp rgb, logistic density
    "act_relu_none": _set(rgb_activation=abi.NSB_ACT_RELU, density_activation=abi.NSB_ACT_NONE),              # raw density: negative alphas and weights
    "linear_colors": _set(linear_colors=1),                                                       # finish without srgb_to_linear
    # render modes
    "ao": _set(render_mode=abi.NSB_RENDER_AO),                                                    # cascade colour and the cell's pcg32 draw
    "distance": _set(render_mode=abi.NSB_RENDER_DISTANCE, depth_scale=0.5),                       # sqrtf(dot3(q, q)) * depth_scale
    "stepsize": _set(render_mode=abi.NSB_RENDER_STEPSIZE),                                        # warp_dt(unwarp_dt(warped dt))
    "depth_scaled": _set(render_mode=abi.NSB_RENDER_DEPTH, depth_scale=2.0),                      # dot3(cam_fwd, q) * depth_scale
    "cost_min_T_0": _set(render_mode=abi.NSB_RENDER_COST, min_transmittance=0.0),                 # step count of rays that never terminate
    "positions_crop": _all(_CROP, _set(render_mode=abi.NSB_RENDER_POSITIONS)),                    # positions of samples inside a crop box
}

# share of pixels each case must hit: about half of what the CPU oracle's 96x54 / 97x55 frame hits (0.76 at the base camera)
MIN_HIT = {name: 0.4 for name in CASES}
MIN_HIT.update({"outside_box": 0.3, "crop_outside": 0.15, "positions_crop": 0.15, "crop_inside": 0.25, "axis_outside": 0.2, "face_plane": 0.2,
                "narrow": 0.9, "cone_1_128": 0.15, "train_not_pow2": 0.3, "act_relu_none": 0.35})

# the cases the fp32-accumulator policy repeats against the reference: the activation, transmittance and linear_colors paths
FP32_CASES = [n for n in CASES if n.startswith(("act_", "min_T_")) or n == "linear_colors"]


def _depth_scale_round_trips(f) -> bool:
    """The reference is handed dataset.scale = 1 / depth_scale and inverts it again (fp32): a value that does not survive the round trip
    would show as a false mismatch."""
    ds = np.float32(f.depth_scale)
    return np.float32(1.0) / (np.float32(1.0) / ds) == ds


def frame(model, name) -> abi.NsbFrame:
    f = syn.make_frame(model, BASE_CAMERA, W, H)
    CASES[name](f)
    return f


# Fields that only the composite and the shading read: cases that differ in nothing else march the same samples
COMPOSITE_FIELDS = ("min_transmittance", "rgb_activation", "density_activation", "linear_colors", "render_mode", "depth_scale")


def _march_key(name):
    g = frame(types.SimpleNamespace(aabb_min=FOX_MIN, aabb_max=FOX_MAX, aabb_scale=syn.FOX_AABB_SCALE), name)
    for k in COMPOSITE_FIELDS:
        setattr(g, k, 0)
    return bytes(g)


def _first_of_each_march():
    seen, out = set(), []
    for n in CASES:
        k = _march_key(n)
        if k not in seen:
            seen.add(k)
            out.append(n)
    return out


# the first case of each distinct march: the reference's sample streams are compared (and stored) once per march, not once per case
MARCH_CASES = _first_of_each_march()


# every depth_scale of the table survives the reference's round trip
for _name, _edit in CASES.items():
    _f = abi.NsbFrame()
    _f.depth_scale = 1.0 / 0.33
    _edit(_f)
    assert _depth_scale_round_trips(_f), (_name, _f.depth_scale)


def camera_outside_render_box(f) -> bool:
    o = np.array([f.camera0[9], f.camera0[10], f.camera0[11]], np.float32)
    mn, mx = np.array(list(f.render_aabb_min), np.float32), np.array(list(f.render_aabb_max), np.float32)
    return bool((o < mn).any() or (o > mx).any())


def pixels(f, n=250, seed=0):
    """A seeded sample of n pixels (all of them on smaller frames), sorted."""
    N = f.width * f.height
    return np.sort(np.random.default_rng(seed).choice(N, min(n, N), replace=False)).astype(np.uint32)
