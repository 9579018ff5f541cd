"""ctypes mirror of include/nerfshop_b200.h (the C ABI) and the loader of the CUDA library.

The product path has NO CPU fallback: `load_library()` raises if the sm_90a shared
library has not been built (`python -c "import __graft_entry__ as g; g.build()"`).
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libnerfshop_b200.so")

NSB_ABI_VERSION = 9
NSB_MLP_ACC_F32, NSB_MLP_ACC_F16 = 0, 1
NSB_NERF_GRIDSIZE = 128
NSB_NERF_CASCADES = 5
NSB_GRID_CELLS = NSB_NERF_CASCADES * NSB_NERF_GRIDSIZE ** 3
NSB_BITFIELD_BYTES = NSB_GRID_CELLS // 8
NSB_GRID_UPDATE_MAX_SAMPLES = 1 << 31

NSB_OK, NSB_ERR_INVALID, NSB_ERR_CUDA, NSB_ERR_STATE, NSB_ERR_UNSUPPORTED = range(5)

NSB_RENDER_AO = 0
NSB_RENDER_SHADE = 1
NSB_RENDER_POSITIONS = 3
NSB_RENDER_DEPTH = 4
NSB_RENDER_DISTANCE = 5
NSB_RENDER_STEPSIZE = 6
NSB_RENDER_DISTORTION = 7
NSB_RENDER_COST = 8
NSB_CAMERA_DISTORTION_NONE, NSB_CAMERA_DISTORTION_ITERATIVE, NSB_CAMERA_DISTORTION_FTHETA = range(3)

NSB_ACT_NONE, NSB_ACT_RELU, NSB_ACT_LOGISTIC, NSB_ACT_EXPONENTIAL = range(4)
NSB_OP_CAGE, NSB_OP_AFFINE = 0, 1

f32 = C.c_float
i32 = C.c_int32
u32 = C.c_uint32
u64 = C.c_uint64


class NsbModelDesc(C.Structure):
    _fields_ = [
        ("n_levels", u32), ("n_features_per_level", u32), ("log2_hashmap_size", u32), ("base_resolution", u32),
        ("per_level_scale", f32), ("n_neurons", u32), ("n_hidden_density", u32), ("n_hidden_rgb", u32), ("sh_degree", u32),
    ]


class NsbFrame(C.Structure):
    _fields_ = [
        ("width", i32), ("height", i32),
        ("focal_length", f32 * 2), ("screen_center", f32 * 2),
        ("camera0", f32 * 12), ("camera1", f32 * 12), ("rolling_shutter", f32 * 4),
        ("render_aabb_min", f32 * 3), ("render_aabb_max", f32 * 3),
        ("train_aabb_min", f32 * 3), ("train_aabb_max", f32 * 3),
        ("cone_angle_constant", f32), ("min_transmittance", f32), ("depth_scale", f32),
        ("rgb_activation", i32), ("density_activation", i32), ("render_mode", i32),
        ("spp_index", u32), ("snap_to_pixel_centers", i32), ("apply_operators", i32),
        ("poisson_target", i32), ("linear_colors", i32), ("min_mip", i32),
        ("tile_rank", i32), ("tile_world", i32), ("show_accel", i32),
        # ABI 3 (all zero = off)
        ("camera_distortion_mode", i32), ("camera_distortion_params", f32 * 7),
        ("dof", f32), ("focus_z", f32),
        ("glow_mode", i32), ("glow_y_cutoff", f32),
        ("envmap_dev", C.c_void_p), ("envmap_resolution", i32 * 2),
        ("distortion_dev", C.c_void_p), ("distortion_resolution", i32 * 2),
    ]


class NsbAffineBox(C.Structure):
    _fields_ = [("min", f32 * 3), ("u", f32 * 3), ("v", f32 * 3), ("w", f32 * 3), ("center", f32 * 3)]


class NsbEditOp(C.Structure):
    _fields_ = [
        ("type", i32),
        ("copy", i32), ("apply_poisson", i32), ("residual_amplitude", f32),
        ("scene_aabb_min", f32 * 3), ("scene_aabb_max", f32 * 3),
        ("bbox_min", f32 * 3), ("bbox_max", f32 * 3),
        ("warped_bbox_min", f32 * 3), ("warped_bbox_max", f32 * 3),
        ("original_warped_bbox_min", f32 * 3), ("original_warped_bbox_max", f32 * 3),
        ("n_tets", u32), ("n_vertices", u32), ("n_lut_idx", u32),
        ("tet_lut_offsets", C.POINTER(u32)), ("tet_lut_idx", C.POINTER(u32)), ("tets", C.POINTER(u32)),
        ("vertices", C.POINTER(f32)), ("original_vertices", C.POINTER(f32)), ("local_rotations", C.POINTER(f32)),
        ("original_bitfield", C.POINTER(C.c_uint8)),
        ("boundary_shs", C.POINTER(f32)), ("boundary_outside_density", C.POINTER(f32)), ("boundary_residual_density", C.POINTER(f32)),
        ("selection_box", NsbAffineBox), ("destination_box", NsbAffineBox),
        ("translation", f32 * 3), ("scale", f32 * 3), ("rotation", f32 * 9),
        ("hide_original", i32), ("correct_dir", i32),
    ]


NSB_COLOR_LINEAR, NSB_COLOR_SRGB, NSB_COLOR_VISPOSNEG = range(3)
NSB_TONEMAP_IDENTITY, NSB_TONEMAP_ACES, NSB_TONEMAP_HABLE, NSB_TONEMAP_REINHARD = range(4)


class NsbTonemap(C.Structure):
    _fields_ = [
        ("color_space", i32), ("output_color_space", i32), ("tonemap_curve", i32), ("clamp_output_color", i32),
        ("exposure", f32), ("background_color", f32 * 4),
    ]


class NsbGridUpdate(C.Structure):
    """Arguments of Testbed::update_density_grid_nerf_operator (testbed_nerf.cu:3533-3639)."""
    _fields_ = [
        ("n_uniform_samples", u32), ("n_nonuniform_samples", u32), ("reset_grid", i32), ("n_cascades", i32),
        ("decay", f32), ("ema_step", u32), ("rng_state", u64), ("rng_inc", u64),
        ("train_aabb_min", f32 * 3), ("train_aabb_max", f32 * 3), ("density_activation", i32), ("apply_operators", i32),
    ]


class NsbBoundarySampling(C.Structure):
    """Members read by GrowingSelection::compute_poisson_boundary (growing_selection.cu:2220-2348)."""
    _fields_ = [
        ("sampling_width", u32), ("hemisphere_width", u32), ("seed", u64),
        ("train_aabb_min", f32 * 3), ("train_aabb_max", f32 * 3), ("rgb_activation", i32), ("density_activation", i32), ("is_inside", i32),
    ]


class NsbRenderStats(C.Structure):
    _fields_ = [
        ("n_rays", u64), ("n_rays_alive", u64), ("n_hit", u64), ("n_samples", u64), ("n_old_samples", u64),
        ("n_kernel_launches", u32), ("gpu_ms", f32), ("fused_ms", f32),
    ]


class NsbGridQuery(C.Structure):
    """Arguments of Testbed::get_density_on_grid (testbed_nerf.cu:4538-4586) in NeRF mode."""
    _fields_ = [("res", i32 * 3), ("aabb_min", f32 * 3), ("aabb_max", f32 * 3), ("train_aabb_min", f32 * 3), ("train_aabb_max", f32 * 3)]


class NsbMeshOptimise(C.Structure):
    """The members of Testbed::m_mesh that Testbed::optimise_mesh_step (testbed_nerf.cu:4470-4513) reads."""
    _fields_ = [("thresh", f32), ("smooth_amount", f32), ("density_amount", f32), ("inflate_amount", f32),
                ("train_aabb_min", f32 * 3), ("train_aabb_max", f32 * 3)]


# every symbol include/nerfshop_b200.h declares (tests/test_abi.py checks the .so exports all of them)
EXPORTED_SYMBOLS = [
    "nsb_abi_version", "nsb_last_error", "nsb_create", "nsb_destroy",
    "nsb_model_n_params", "nsb_set_mlp_accumulator", "nsb_upload_model", "nsb_upload_model_dev", "nsb_upload_occupancy_dev", "nsb_upload_occupancy", "nsb_upload_density_grid", "nsb_set_edit_ops",
    "nsb_update_density_grid", "nsb_download_density_grid", "nsb_cage_attach_mvc", "nsb_cage_deform", "nsb_cage_download", "nsb_cage_vanish",
    "nsb_poisson_boundary", "nsb_cage_set_membrane",
    "nsb_render", "nsb_render_host", "nsb_render_host_async", "nsb_host_frame_wait", "nsb_get_stats", "nsb_debug_counters",
    "nsb_tiles_for_rank", "nsb_pack_tiles", "nsb_unpack_tiles", "nsb_unpack_gathered", "nsb_accumulate", "nsb_tonemap",
    "nsb_inference", "nsb_density", "nsb_encode", "nsb_map_rays", "nsb_poisson_residuals", "nsb_map_rays_op", "nsb_poisson_residuals_op",
    "nsb_map_positions", "nsb_poisson_residual_density", "nsb_march_trace",
    "nsb_build_tet_grid", "nsb_compute_mvc", "nsb_interpolate_with_mvc", "nsb_local_rotations",
    "nsb_density_on_grid", "nsb_marching_cubes", "nsb_mesh_shade", "nsb_mesh_download",
    "nsb_density_gradient", "nsb_mesh_optimise",
    "nsb_rgba_on_grid", "nsb_density_png_extent", "nsb_density_png", "nsb_rgba_png",
    "nsb_render_accumulate", "nsb_frame_to_rgba8",
    "nsb_reference_image", "nsb_image_metrics",
]

_lib = None


class NsbError(RuntimeError):
    pass


def load_library(path: str | None = None) -> C.CDLL:
    """Loads libnerfshop_b200.so. Fails loudly when it is missing — there is no CPU fallback."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or os.environ.get("NSB_LIB_PATH") or LIB_PATH  # NSB_LIB_PATH: A/B builds of the same library
    if not os.path.exists(p):
        raise NsbError(
            f"{p} not found: build the sm_90a extension first (python -c 'import __graft_entry__ as g; g.build()'). "
            "nerfshop_b200 has no CPU fallback."
        )
    lib = C.CDLL(p)
    lib.nsb_last_error.restype = C.c_char_p
    lib.nsb_abi_version.restype = C.c_int
    if lib.nsb_abi_version() != NSB_ABI_VERSION:
        raise NsbError(f"ABI mismatch: library {lib.nsb_abi_version()} vs bindings {NSB_ABI_VERSION}")
    vp = C.c_void_p
    lib.nsb_create.argtypes = [C.c_int, C.POINTER(vp)]
    lib.nsb_destroy.argtypes = [vp]
    lib.nsb_model_n_params.argtypes = [C.POINTER(NsbModelDesc), C.POINTER(u64)]
    lib.nsb_upload_model.argtypes = [vp, C.POINTER(NsbModelDesc), vp, u64]
    lib.nsb_set_mlp_accumulator.argtypes = [vp, i32]
    lib.nsb_upload_model_dev.argtypes = [vp, C.POINTER(NsbModelDesc), vp, u64]
    lib.nsb_upload_occupancy_dev.argtypes = [vp, vp, u64]
    lib.nsb_map_rays_op.argtypes = [vp, i32, vp, vp, u32, vp]
    lib.nsb_poisson_residuals_op.argtypes = [vp, i32, vp, u32, vp, vp, vp, vp]
    lib.nsb_map_positions.argtypes = [vp, i32, vp, u32, vp, u32, vp]
    lib.nsb_poisson_residual_density.argtypes = [vp, i32, vp, u32, vp, u32, vp]
    lib.nsb_upload_occupancy.argtypes = [vp, vp, u64]
    lib.nsb_upload_density_grid.argtypes = [vp, vp, u64, vp]
    lib.nsb_update_density_grid.argtypes = [vp, C.POINTER(NsbGridUpdate), vp]
    lib.nsb_download_density_grid.argtypes = [vp, vp, vp]
    lib.nsb_cage_attach_mvc.argtypes = [vp, i32, vp, u32]
    lib.nsb_cage_deform.argtypes = [vp, i32, vp, u32, vp]
    lib.nsb_cage_download.argtypes = [vp, i32, vp, vp, vp, vp, u64, C.POINTER(u64), vp]
    lib.nsb_cage_vanish.argtypes = [vp, i32, C.POINTER(u64), vp]
    lib.nsb_poisson_boundary.argtypes = [vp, vp, u32, C.POINTER(NsbBoundarySampling), vp, vp]
    lib.nsb_cage_set_membrane.argtypes = [vp, i32, vp, u32, vp, vp, vp, vp, f32, i32, vp, vp, vp]
    lib.nsb_set_edit_ops.argtypes = [vp, C.POINTER(NsbEditOp), i32]
    lib.nsb_render.argtypes = [vp, C.POINTER(NsbFrame), vp, vp, vp]
    lib.nsb_render_host.argtypes = [vp, C.POINTER(NsbFrame), vp, vp]
    lib.nsb_render_host_async.argtypes = [vp, C.POINTER(NsbFrame), vp, vp, C.POINTER(u64)]
    lib.nsb_host_frame_wait.argtypes = [vp, u64]
    lib.nsb_get_stats.argtypes = [vp, C.POINTER(NsbRenderStats)]
    lib.nsb_debug_counters.argtypes = [vp, C.POINTER(u64), i32]
    lib.nsb_tiles_for_rank.argtypes = [i32, i32, i32, i32, C.POINTER(u32)]
    lib.nsb_pack_tiles.argtypes = [vp, vp, vp, i32, i32, i32, i32, vp, vp, vp]
    lib.nsb_unpack_tiles.argtypes = [vp, vp, vp, i32, i32, i32, i32, vp, vp, vp]
    lib.nsb_unpack_gathered.argtypes = [vp, vp, vp, i32, i32, i32, i32, C.c_uint32, vp, vp, vp]
    lib.nsb_accumulate.argtypes = [vp, vp, vp, i32, i32, u32, i32, vp]
    lib.nsb_tonemap.argtypes = [vp, vp, vp, i32, i32, C.POINTER(NsbTonemap), vp]
    lib.nsb_inference.argtypes = [vp, vp, u32, vp, u32, vp]
    lib.nsb_density.argtypes = [vp, vp, u32, vp, u32, vp]
    lib.nsb_encode.argtypes = [vp, vp, u32, vp, u32, vp]
    lib.nsb_map_rays.argtypes = [vp, vp, vp, u32, vp]
    lib.nsb_poisson_residuals.argtypes = [vp, vp, u32, vp, vp, vp, vp]
    lib.nsb_march_trace.argtypes = [vp, C.POINTER(NsbFrame), vp, u32, u32, vp, vp, vp, vp]
    lib.nsb_build_tet_grid.argtypes = [vp, u32, vp, u32, vp, vp, u64, C.POINTER(u64), vp]
    lib.nsb_compute_mvc.argtypes = [vp, u32, vp, u32, vp, u32, f32, vp]
    lib.nsb_interpolate_with_mvc.argtypes = [vp, u32, u32, vp, vp]
    lib.nsb_local_rotations.argtypes = [vp, vp, vp, u32, vp]
    lib.nsb_density_on_grid.argtypes = [vp, C.POINTER(NsbGridQuery), vp, vp]
    lib.nsb_marching_cubes.argtypes = [vp, vp, C.POINTER(i32), C.POINTER(f32), C.POINTER(f32), f32, C.POINTER(u64), C.POINTER(u64), vp]
    lib.nsb_mesh_shade.argtypes = [vp, C.POINTER(f32), C.POINTER(f32), i32, i32, vp]
    lib.nsb_mesh_download.argtypes = [vp, vp, vp, vp, u64, vp, u64]
    lib.nsb_density_gradient.argtypes = [vp, vp, u32, vp, u32, vp, vp, u32, vp]
    lib.nsb_mesh_optimise.argtypes = [vp, C.POINTER(NsbMeshOptimise), u32, vp]
    lib.nsb_rgba_on_grid.argtypes = [vp, C.POINTER(NsbGridQuery), C.POINTER(f32), i32, i32, vp, vp]
    lib.nsb_density_png_extent.argtypes = [C.POINTER(i32), i32, C.POINTER(u32), C.POINTER(u32)]
    lib.nsb_density_png.argtypes = [vp, vp, C.POINTER(i32), f32, f32, i32, vp, vp, vp]
    lib.nsb_rgba_png.argtypes = [vp, vp, C.POINTER(i32), i32, vp, vp]
    lib.nsb_render_accumulate.argtypes = [vp, C.POINTER(NsbFrame), u32, C.POINTER(NsbTonemap), vp, vp, vp]
    lib.nsb_frame_to_rgba8.argtypes = [vp, vp, i32, i32, f32, i32, vp, vp]
    lib.nsb_reference_image.argtypes = [vp, vp, i32, i32, i32, i32, C.POINTER(f32), vp, vp]
    lib.nsb_image_metrics.argtypes = [vp, vp, vp, i32, i32, vp, vp, vp, vp]
    for name in EXPORTED_SYMBOLS:
        fn = getattr(lib, name)
        if name not in ("nsb_last_error", "nsb_abi_version"):
            fn.restype = C.c_int
    if path is None:
        _lib = lib
    return lib


def check(lib: C.CDLL, status: int, what: str) -> None:
    if status != NSB_OK:
        msg = lib.nsb_last_error()
        raise NsbError(f"{what} failed (status {status}): {msg.decode() if msg else ''}")
