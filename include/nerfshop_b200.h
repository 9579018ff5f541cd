/*
 * nerfshop_b200.h — C ABI of the H100-native NeRFshop render path.
 *
 * This is the drop-in boundary for ONE hot path of graphdeco-inria/nerfshop:
 *   Testbed::render_nerf            (reference src/testbed_nerf.cu:3066-3201)
 *     -> NerfTracer::init_rays_from_camera (:2683-2756)
 *     -> NerfTracer::trace                 (:2772-3002)
 *     -> shade_kernel_nerf                 (:2448-2483)
 * together with the three class surfaces it is called through:
 *   NerfNetwork<T>   (include/neural-graphics-primitives/nerf_network.h:87-120)
 *   EditOperator     (include/neural-graphics-primitives/editing/edit_operator.h:25-94)
 *   Testbed::NerfTracer (include/neural-graphics-primitives/testbed.h:129-240)
 *
 * The reference has no FFI; its boundary is C++ classes. Every entry point
 * below names the reference member it replaces. A C++ shim that keeps the
 * reference's class names on top of this ABI is in nerfshop_b200/host/.
 *
 * Conventions
 *  - plain pointers and sizes only; no exceptions cross the ABI; every call
 *    returns an NsbStatus and nsb_last_error() gives the message. After a
 *    call fails with NSB_ERR_CUDA because an allocation failed, the context
 *    can still be used, and any model or operator it reports is intact.
 *  - "host" pointers are read during the call and never retained.
 *  - "dev" pointers are CUDA device pointers owned by the caller.
 *  - matrices are column-major like Eigen (camera 3x4: 12 floats, col 0..3).
 *  - one context per device; calls on one context are serialised by the caller
 *    (same contract as the reference: everything runs on m_inference_stream).
 */
#ifndef NERFSHOP_B200_H
#define NERFSHOP_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NSB_ABI_VERSION 7

/* reference: common_nerf.h:16-39 */
#define NSB_NERF_GRIDSIZE 128u
#define NSB_NERF_CASCADES 5u
#define NSB_GRID_CELLS (NSB_NERF_CASCADES * NSB_NERF_GRIDSIZE * NSB_NERF_GRIDSIZE * NSB_NERF_GRIDSIZE)
#define NSB_BITFIELD_BYTES (NSB_GRID_CELLS / 8u) /* 1,310,720 */

typedef enum {
	NSB_OK = 0,
	NSB_ERR_INVALID = 1,     /* bad argument / unsupported configuration */
	NSB_ERR_CUDA = 2,        /* a CUDA call failed (message has the CUDA error) */
	NSB_ERR_STATE = 3,       /* call order: model / occupancy not uploaded yet */
	NSB_ERR_UNSUPPORTED = 4  /* feature of the reference that this path does not cover */
} NsbStatus;

/* reference: common.h:71-84 (ERenderMode); only the modes that do not need
 * network input gradients are covered. */
typedef enum {
	NSB_RENDER_AO = 0,
	NSB_RENDER_SHADE = 1,
	NSB_RENDER_POSITIONS = 3,
	NSB_RENDER_DEPTH = 4,
	NSB_RENDER_DISTANCE = 5,
	NSB_RENDER_STEPSIZE = 6,
	NSB_RENDER_DISTORTION = 7, /* the distortion map itself, written by ray initialisation (testbed_nerf.cu:2596-2607) */
	NSB_RENDER_COST = 8
} NsbRenderMode;

/* reference: common.h:107-112 (ENerfActivation) */
typedef enum {
	NSB_ACT_NONE = 0,
	NSB_ACT_RELU = 1,
	NSB_ACT_LOGISTIC = 2,
	NSB_ACT_EXPONENTIAL = 3
} NsbActivation;

typedef struct NsbContext NsbContext;

/* Network configuration = configs/nerf/base.json + the values Testbed::reset_network
 * derives (testbed.cu:2258-2292). Only the base.json topology is implemented:
 * HashGrid F=2 -> 64x1 density MLP (16 out) -> SH deg 4 -> 64x2 rgb MLP (3 out, padded 16). */
typedef struct {
	uint32_t n_levels;            /* 16 */
	uint32_t n_features_per_level;/* 2  */
	uint32_t log2_hashmap_size;   /* 19 */
	uint32_t base_resolution;     /* 16 */
	float    per_level_scale;     /* exp(ln(2048*aabb_scale/16)/15); fox: 1.5157166 */
	uint32_t n_neurons;           /* 64 */
	uint32_t n_hidden_density;    /* 1  */
	uint32_t n_hidden_rgb;        /* 2  */
	uint32_t sh_degree;           /* 4  */
} NsbModelDesc;

/* Per-frame inputs = the arguments of Testbed::render_nerf (testbed.h:305) plus the
 * Testbed members it reads (testbed_nerf.cu:3082-3138). */
typedef struct {
	int32_t  width, height;            /* render_buffer.in_resolution() */
	float    focal_length[2];          /* pixels */
	float    screen_center[2];
	float    camera0[12];              /* 3x4 column-major */
	float    camera1[12];
	float    rolling_shutter[4];
	float    render_aabb_min[3], render_aabb_max[3]; /* m_render_aabb */
	float    train_aabb_min[3],  train_aabb_max[3];  /* m_aabb */
	float    cone_angle_constant;      /* m_nerf.cone_angle_constant */
	float    min_transmittance;        /* m_nerf.rendering_min_transmittance (0.01) */
	float    depth_scale;              /* 1 / dataset.scale */
	int32_t  rgb_activation;           /* NsbActivation */
	int32_t  density_activation;       /* NsbActivation */
	int32_t  render_mode;              /* NsbRenderMode */
	uint32_t spp_index;                /* render_buffer.spp() */
	int32_t  snap_to_pixel_centers;
	int32_t  apply_operators;          /* m_enable_edits && !m_distill */
	int32_t  poisson_target;           /* NerfTracer::m_poisson_target */
	int32_t  linear_colors;            /* m_nerf.training.linear_colors */
	int32_t  min_mip;                  /* (show_accel>=0) ? show_accel : 0: the coarsest occupancy cascade the march may test (:2750, :2849) */
	/* image-plane partition (new; the reference is single-GPU): this context renders the
	 * 16x8-pixel tiles whose linear index t satisfies t % tile_world == tile_rank. */
	int32_t  tile_rank, tile_world;
	/* m_nerf.show_accel >= 0 (the GUI's occupancy-grid visualisation): 0 = off (the reference's -1); 1 = on with show_accel = min_mip: every sample's
	 * alpha is forced to 1 (testbed_nerf.cu:788-790) and Positions mode colours the occupancy cells (:913-923). Zero-initialised frames have it off. */
	int32_t  show_accel;
	/* ---- ABI 3: the remaining arguments of init_rays_with_payload_kernel_nerf / pixel_to_ray / composite_kernel_nerf. All zero = off. ---- */
	/* m_nerf.render_with_camera_distortion ? m_nerf.render_distortion : CameraDistortion{} (testbed_nerf.cu:3081,3096; common.h:166-175;
	 * pixel_to_ray common_device.cuh:263-277): NsbCameraDistortionMode; params = {k1, k2, p1, p2} (iterative OpenCV undistortion, :163-197)
	 * or {r0..r4, res_x, res_y} (f-theta, :232-245) */
	int32_t  camera_distortion_mode;
	float    camera_distortion_params[7];
	/* depth of field (pixel_to_ray :285-294): dof = m_dof (aperture), focus_z = m_slice_plane_z + m_scale (> 0; the Slice side path, which the
	 * reference selects with a negative plane_z, is not covered). dof == 0: pinhole, focus_z unused. */
	float    dof;
	float    focus_z;
	/* m_nerf.m_glow_mode / m_glow_y_cutoff (composite_kernel_nerf :807-903): bit 0 green grid, 1 cut line, 2 mask to alpha, 3 radial, 4 grid mode */
	int32_t  glow_mode;
	float    glow_y_cutoff;
	/* m_envmap (init_rays :2581-2583, envmap.cuh:30-62): float RGBA texels in DEVICE memory, row-major [res_y][res_x][4]; when set, every pixel of
	 * the frame buffer is first overwritten with the environment colour of its ray (the frame is then blended over it). NULL: the buffer is kept. */
	const float* envmap_dev;
	int32_t  envmap_resolution[2];
	/* m_distortion.map (pixel_to_ray :278-280, read_image common_device.cuh:79-110): float2 texels in DEVICE memory added to the camera-space ray
	 * direction; also what NSB_RENDER_DISTORTION visualises (init_rays :2596-2607). NULL: none. */
	const float* distortion_dev;
	int32_t  distortion_resolution[2];
} NsbFrame;

/* reference: common.h:166-170 (ECameraDistortionMode) */
typedef enum { NSB_CAMERA_DISTORTION_NONE = 0, NSB_CAMERA_DISTORTION_ITERATIVE = 1, NSB_CAMERA_DISTORTION_FTHETA = 2 } NsbCameraDistortionMode;

typedef enum { NSB_OP_CAGE = 0, NSB_OP_AFFINE = 1 } NsbEditOpType;

/* Oriented box of affine_bounding_box.cuh:88-93 (only the fields contains() reads + center). */
typedef struct {
	float min[3], u[3], v[3], w[3], center[3];
} NsbAffineBox;

/* One EditOperator as the POD of its device-kernel arguments.
 *  cage  : interpolate_tet (cage_deformation.cu:197-212) + compute_residual_poisson_kernel (:431-456)
 *  affine: translate_in_box (affine_duplication.cu:92-102)
 * All pointers are HOST pointers; nsb_set_edit_ops copies them to the device. */
typedef struct {
	int32_t type; /* NsbEditOpType */

	/* ---- cage ---- */
	int32_t copy;               /* GrowingSelection::m_copy */
	int32_t apply_poisson;      /* CageDeformation::m_apply_poisson */
	float   residual_amplitude; /* CageDeformation::m_residual_amplitude */
	float   scene_aabb_min[3], scene_aabb_max[3];                 /* m_scene_aabb */
	float   bbox_min[3], bbox_max[3];                             /* TetMesh::bbox (deformed, world) */
	float   warped_bbox_min[3], warped_bbox_max[3];               /* TetMesh::warped_bbox */
	float   original_warped_bbox_min[3], original_warped_bbox_max[3]; /* TetMesh::original_warped_bbox */
	uint32_t n_tets, n_vertices, n_lut_idx;
	const uint32_t* tet_lut_offsets;   /* [NSB_GRID_CELLS + 1] CSR offsets, cell = mip*128^3 + morton */
	const uint32_t* tet_lut_idx;       /* [n_lut_idx] */
	const uint32_t* tets;              /* [4*n_tets] */
	const float*    vertices;          /* [3*n_vertices] deformed */
	const float*    original_vertices; /* [3*n_vertices] canonical */
	const float*    local_rotations;   /* [9*n_tets] column-major, or NULL */
	const uint8_t*  original_bitfield; /* [NSB_BITFIELD_BYTES] */
	const float*    boundary_shs;              /* [27*n_vertices] SH9RGB column-major (9 x 3), or NULL */
	const float*    boundary_outside_density;  /* [n_vertices] or NULL */
	const float*    boundary_residual_density; /* [n_vertices] or NULL */
	/* The render's membrane residuals use an operator only when all three boundary arrays are given; the density-grid residual
	 * (nsb_poisson_residual_density, the occupancy update) needs only boundary_residual_density. */

	/* ---- affine ---- */
	NsbAffineBox selection_box;    /* m_warped_selection_box */
	NsbAffineBox destination_box;  /* m_warped_destination_box */
	float   translation[3];        /* m_warped_translation */
	float   scale[3];              /* m_scale */
	float   rotation[9];           /* m_rotation_matrix, column-major */
	int32_t hide_original;         /* m_hide_original */
	int32_t correct_dir;           /* m_correct_dir */
} NsbEditOp;

/* Counters of the last nsb_render call (the reference logs the same in ERenderMode::Cost,
 * testbed_nerf.cu:3190-3200). */
typedef struct {
	uint64_t n_rays;          /* rays generated by this context (its tiles) */
	uint64_t n_rays_alive;    /* rays that entered the render AABB */
	uint64_t n_hit;           /* rays shaded into the framebuffer (A > 0.001) */
	uint64_t n_samples;       /* network evaluations (occupied samples composited or masked) */
	uint64_t n_old_samples;   /* extra density evaluations for the membrane target */
	uint32_t n_kernel_launches;
	float    gpu_ms;          /* device time of the whole call (both kernels + counters reset), CUDA events on the launch stream */
	float    fused_ms;        /* device time of k_render_fused alone */
} NsbRenderStats;

/* ---- lifetime -------------------------------------------------------------------- */
int         nsb_abi_version(void);
const char* nsb_last_error(void);
/* device < 0: current device. */
NsbStatus   nsb_create(int device, NsbContext** out);
NsbStatus   nsb_destroy(NsbContext* ctx);

/* ---- state uploads (host pointers) ------------------------------------------------- */
/* Number of fp16 parameters the description implies, in the reference's block order
 * [density MLP][rgb MLP][hash grid] (nerf_network_full.h:316-349). */
NsbStatus nsb_model_n_params(const NsbModelDesc* desc, uint64_t* n_params);
/* replaces tcnn::Trainer::deserialize -> NerfNetwork::set_params (testbed.cu:3087). */
NsbStatus nsb_upload_model(NsbContext* ctx, const NsbModelDesc* desc, const uint16_t* params_fp16, uint64_t n_params);
/* Accumulator policy of the two fully fused MLPs (every entry point that evaluates the network). The reference's tiny-cuda-nn FullyFusedMLP
 * runs wmma m16n16k16 with __half accumulator fragments (SURVEY.md Appendix B; the submodule is absent, so this is not verifiable here):
 *   NSB_MLP_ACC_F16 (default) fp16 accumulators: the running sum is rounded to fp16 by every K=16 wgmma, as with __half fragments;
 *   NSB_MLP_ACC_F32 fp32 accumulators, one rounding to fp16 per layer output (more accurate, not what the reference computes).
 * The two differ by up to 1e-2 in RGBA on 0.02 % of the pixels of a 480x270 frame (tests/test_mlp_policy.py, DESIGN.md section 3). */
typedef enum { NSB_MLP_ACC_F32 = 0, NSB_MLP_ACC_F16 = 1 } NsbMlpAccumulator;
NsbStatus nsb_set_mlp_accumulator(NsbContext* ctx, int32_t policy);
/* replaces Testbed::Nerf::density_grid_bitfield (testbed.h:626; built at testbed.cu:3079). */
NsbStatus nsb_upload_occupancy(NsbContext* ctx, const uint8_t* bitfield, uint64_t n_bytes);
/* replaces Testbed::update_density_grid_mean_and_bitfield (testbed_nerf.cu:3642-3658: mean of cascade 0, grid_to_bitfield :514,
 * bitfield_max_pool :534), the step load_snapshot runs on the float density grid of a snapshot (testbed.cu:3078-3079):
 * density_grid: HOST float[5*128^3]; the resulting bitfield becomes the context's occupancy and, if bitfield_out != NULL,
 * is also copied back (NSB_BITFIELD_BYTES). */
NsbStatus nsb_upload_density_grid(NsbContext* ctx, const float* density_grid, uint64_t n_floats, uint8_t* bitfield_out);
/* The same two uploads from DEVICE memory (the reference owns both on the device: tcnn::Trainer::params(), Testbed::Nerf::density_grid_bitfield):
 * the 26 MB hash table is copied device-to-device; only the 20 KB of MLP weights pass through the host to be laid out as tensor-core operands. */
NsbStatus nsb_upload_model_dev(NsbContext* ctx, const NsbModelDesc* desc, const uint16_t* params_fp16_dev, uint64_t n_params);
NsbStatus nsb_upload_occupancy_dev(NsbContext* ctx, const uint8_t* bitfield_dev, uint64_t n_bytes);
/* replaces NerfTracer::{add,delete,reset}_edit_operator; list order = m_edit_operators order
 * (operators are applied in REVERSE list order, testbed_nerf.cu:2868,2899). n = 0 clears. */
NsbStatus nsb_set_edit_ops(NsbContext* ctx, const NsbEditOp* ops, int32_t n);

/* ---- the hot path -------------------------------------------------------------------- */
/* replaces Testbed::render_nerf. fb_dev: float4[width*height] (render_buffer.frame_buffer()),
 * depth_dev: float[width*height] (depth_buffer()). Like the reference, pixels that hit are
 * over-blended onto what fb_dev already holds; depth is set to 1e10 for every generated ray.
 * Stream-ordered on `stream` (a cudaStream_t, may be NULL); returns without synchronising. */
NsbStatus nsb_render(NsbContext* ctx, const NsbFrame* frame, float* fb_dev, float* depth_dev, void* stream);
/* Same through HOST buffers (the reference's Testbed::render_to_cpu recipe, python_api.cu:129-175):
 * clears a device framebuffer, renders, copies RGBA (+depth if non-NULL) back, synchronises. */
NsbStatus nsb_render_host(NsbContext* ctx, const NsbFrame* frame, float* fb_host, float* depth_host);
/* The same without the wait (new; the reference's render_to_cpu is synchronous): the frame is rendered into one of two device framebuffers the
 * context owns and copied back on a second stream, so the copy of frame k (41.5 MB at 1080p) overlaps the render of frame k+1. Returns a ticket;
 * fb_host / depth_host (pinned memory, or the copy is not asynchronous) belong to the library until nsb_host_frame_wait(ticket) returns. At most
 * two frames are in flight: a third call waits for the oldest copy. */
NsbStatus nsb_render_host_async(NsbContext* ctx, const NsbFrame* frame, float* fb_host, float* depth_host, uint64_t* ticket);
NsbStatus nsb_host_frame_wait(NsbContext* ctx, uint64_t ticket);
/* Synchronises and returns the counters of the last render. */
NsbStatus nsb_get_stats(NsbContext* ctx, NsbRenderStats* out);

/* Diagnostics of the last nsb_render (not part of the reference surface), counted per render tile (128 threads; a CTA of the
 * fused renderer holds 5-7 of them): out[0..6] = MLP rounds summed over tiles, per-phase SM cycles of thread 0 of each tile summed
 * over tiles {acquire/march, encode, mlp, composite, total}, tiles run. */
NsbStatus nsb_debug_counters(NsbContext* ctx, uint64_t* out, int32_t n);

/* Multi-GPU helpers: packed tile buffers for the single framebuffer gather.
 * nsb_tiles_for_rank gives how many 16x8 tiles (and so how many float4 = n_tiles*128) a rank owns. */
NsbStatus nsb_tiles_for_rank(int32_t width, int32_t height, int32_t rank, int32_t world, uint32_t* n_tiles);
/* dst_packed[(local_tile*128 + lane)] <- fb[pixel(tile,lane)] for this rank's tiles. */
NsbStatus nsb_pack_tiles(NsbContext* ctx, const float* fb_dev, const float* depth_dev, int32_t width, int32_t height,
                         int32_t rank, int32_t world, float* dst_packed_rgba_dev, float* dst_packed_depth_dev, void* stream);
/* inverse: scatter one rank's packed tiles into a full framebuffer. */
NsbStatus nsb_unpack_tiles(NsbContext* ctx, const float* src_packed_rgba_dev, const float* src_packed_depth_dev,
                           int32_t width, int32_t height, int32_t rank, int32_t world,
                           float* fb_dev, float* depth_dev, void* stream);

/* inverse for a whole all-gather result, ONE launch: rank k's packed float4 tiles start at gathered_rgba_dev + k*rank_stride_floats, its packed
 * depth floats (gathered_depth_dev may be NULL) at gathered_depth_dev + k*rank_stride_floats — the two arrays may be the two halves of one gathered
 * buffer. Every rank's tiles except skip_rank's (the caller's own, already in fb; -1 scatters all) are written into fb_dev / depth_dev.
 * New (the reference is single-GPU): SURVEY.md section 8e. */
NsbStatus nsb_unpack_gathered(NsbContext* ctx, const float* gathered_rgba_dev, const float* gathered_depth_dev, int32_t width, int32_t height,
                              int32_t skip_rank, int32_t world, uint32_t rank_stride_floats, float* fb_dev, float* depth_dev, void* stream);

/* ---- frame post-process (SURVEY.md §8f-4): what Testbed::render_frame runs right after render_nerf ----------------- */
/* reference: common.h:122-135 */
typedef enum { NSB_COLOR_LINEAR = 0, NSB_COLOR_SRGB = 1, NSB_COLOR_VISPOSNEG = 2 } NsbColorSpace;
typedef enum { NSB_TONEMAP_IDENTITY = 0, NSB_TONEMAP_ACES = 1, NSB_TONEMAP_HABLE = 2, NSB_TONEMAP_REINHARD = 3 } NsbTonemapCurve;
typedef struct {
	int32_t color_space;         /* CudaRenderBuffer::m_color_space */
	int32_t output_color_space;  /* to_srgb ? SRGB : Linear */
	int32_t tonemap_curve;       /* m_tonemap_curve */
	int32_t clamp_output_color;
	float   exposure;            /* stops */
	float   background_color[4]; /* sRGB-encoded, like the reference's m_background_color */
} NsbTonemap;
/* replaces CudaRenderBuffer::accumulate -> accumulate_kernel (render_buffer.cu:217-258, :540-560): running mean over spp;
 * spp = samples already in the accumulate buffer (0: the buffer is overwritten). */
NsbStatus nsb_accumulate(NsbContext* ctx, const float* frame_buffer_dev, float* accumulate_buffer_dev, int32_t width, int32_t height,
                         uint32_t spp, int32_t color_space, void* stream);
/* replaces CudaRenderBuffer::tonemap -> tonemap_kernel (render_buffer.cu:471-499, :262-332): background blend, exposure, curve,
 * output colour space; writes float4[width*height] (the reference writes a CUDA surface of the same content). */
NsbStatus nsb_tonemap(NsbContext* ctx, const float* accumulate_buffer_dev, float* out_rgba_dev, int32_t width, int32_t height,
                      const NsbTonemap* params, void* stream);

/* ---- occupancy update through the edit operators (SURVEY.md §8f-2) ------------------------------------------------ */
/* The arguments Testbed::update_density_grid_nerf_operator (testbed_nerf.cu:3533-3639) takes from Testbed members. */
typedef struct {
	uint32_t n_uniform_samples;    /* n_uniform_density_grid_samples: cells drawn with threshold -0.01 (any trained cell) */
	uint32_t n_nonuniform_samples; /* n_nonuniform_density_grid_samples: cells drawn with threshold NERF_MIN_OPTICAL_THICKNESS */
	int32_t  reset_grid;           /* reset_grid: zero the running grid first (:3558) */
	int32_t  n_cascades;           /* m_nerf.max_cascade + 1 */
	float    decay;                /* m_nerf.training.density_grid_decay (0.95) */
	uint32_t ema_step;             /* m_nerf.density_grid_ema_step BEFORE the call (the host increments it afterwards, :3636) */
	uint64_t rng_state, rng_inc;   /* m_rng (tcnn pcg32) BEFORE the call; the reference advances it by 2^32 after each of the
	                                  two sample-generation launches (:3576,:3589) — the host mirror does the same */
	float    train_aabb_min[3], train_aabb_max[3]; /* m_aabb */
	int32_t  density_activation;   /* NsbActivation */
	int32_t  apply_operators;      /* 0: behave like update_density_grid_nerf's sampling/splat without operators */
} NsbGridUpdate;
/* replaces Testbed::update_density_grid_nerf_operator + update_density_grid_mean_and_bitfield: draws grid samples
 * (generate_grid_samples_nerf_nonuniform, common_nerf.cu:179-208), maps them through the uploaded operators in reverse order
 * (EditOperator::map_positions, :3593-3599), evaluates NerfNetwork::density, activates, adds the membrane residual densities
 * (compute_poisson_residual_density, cage_deformation.cu:341-383), max-splats into a scratch grid (:447-463), merges into the
 * context's running density grid (ema_grid_samples_nerf, :483-506) and rebuilds the occupancy bitfield the renderer marches.
 * The running grid is the one nsb_upload_density_grid stored (all zeros if none was uploaded). Stream-ordered.
 * NSB_ERR_INVALID, before anything is launched, if n_uniform_samples + n_nonuniform_samples exceeds NSB_GRID_UPDATE_MAX_SAMPLES
 * (2^31, over 200 times the reference's largest update, 5 x 128^3). */
#define NSB_GRID_UPDATE_MAX_SAMPLES (1ull << 31)
NsbStatus nsb_update_density_grid(NsbContext* ctx, const NsbGridUpdate* params, void* stream);
/* copies the context's running density grid (HOST float[5*128^3], may be NULL) and occupancy bitfield (HOST, NSB_BITFIELD_BYTES,
 * may be NULL) back; synchronises the device. */
NsbStatus nsb_download_density_grid(NsbContext* ctx, float* density_grid, uint8_t* bitfield);

/* ---- operator-level entry points (unit parity; same device code as nsb_render) ------- */
/* replaces NerfNetwork::inference_mixed_precision (testbed_nerf.cu:2892,2913):
 * coords_dev: n x 7 floats {pos3 (warped), dt, dir3 (warped)} = NerfCoordinate (nerf.h:73);
 * out_dev: fp16, row-major 16 x n_padded (element (k,i) at k*n_padded + i), rows 0-2 rgb raw, row 3 density raw.
 * n_padded = n rounded up to 128 (tcnn::batch_size_granularity). */
NsbStatus nsb_inference(NsbContext* ctx, const float* coords_dev, uint32_t n, uint16_t* out_dev, uint32_t n_padded, void* stream);
/* replaces NerfNetwork::density (nerf_network_full.h:223-239): out_dev fp16 [16 x n_padded] row-major = density MLP output. */
NsbStatus nsb_density(NsbContext* ctx, const float* coords_dev, uint32_t n, uint16_t* out_dev, uint32_t n_padded, void* stream);
/* hash-grid encoding alone (tcnn GridEncoding inference): out_dev fp16 [32 x n_padded] row-major. */
NsbStatus nsb_encode(NsbContext* ctx, const float* coords_dev, uint32_t n, uint16_t* out_dev, uint32_t n_padded, void* stream);
/* replaces the loop over EditOperator::map_rays (testbed_nerf.cu:2896-2904): applies all uploaded
 * operators in reverse order, in place; empty_mask_dev: n bytes (cleared first, like :2898). */
NsbStatus nsb_map_rays(NsbContext* ctx, float* coords_dev, uint8_t* empty_mask_dev, uint32_t n, void* stream);
/* replaces the loop over EditOperator::compute_poisson_full_residuals (:2867-2883) for a flat list of
 * n samples: sh_dev [27*n], out_density_dev [n], residual_density_dev [n] (cleared first, like :2863-2866). */
NsbStatus nsb_poisson_residuals(NsbContext* ctx, const float* coords_dev, uint32_t n,
                                float* sh_dev, float* out_density_dev, float* residual_density_dev, void* stream);
/* ONE operator of the uploaded list (op_index >= 0) = one call of the EditOperator virtual (edit_operator.h:43,45,68,81); outputs are not cleared,
 * like the virtuals. op_index < 0 = the reference's loop over all operators in reverse order with its clears (the two functions above).
 *   nsb_map_rays_op                 EditOperator::map_rays                          (interpolate_tet / translate_in_box)
 *   nsb_poisson_residuals_op        EditOperator::compute_poisson_full_residuals   (compute_residual_poisson_kernel)
 *   nsb_map_positions               EditOperator::map_positions                    (interpolate_tet_pos / translate_in_box_pos; PitchedPtr<NerfPosition>: stride in floats)
 *   nsb_poisson_residual_density    EditOperator::compute_poisson_residual_density (density_fp16[i] += (half) interpolated residual density) */
NsbStatus nsb_map_rays_op(NsbContext* ctx, int32_t op_index, float* coords_dev, uint8_t* empty_mask_dev, uint32_t n, void* stream);
NsbStatus nsb_poisson_residuals_op(NsbContext* ctx, int32_t op_index, const float* coords_dev, uint32_t n, float* sh_dev, float* out_density_dev,
                                   float* residual_density_dev, void* stream);
NsbStatus nsb_map_positions(NsbContext* ctx, int32_t op_index, float* positions_dev, uint32_t stride_floats, uint8_t* empty_mask_dev, uint32_t n, void* stream);
NsbStatus nsb_poisson_residual_density(NsbContext* ctx, int32_t op_index, const float* positions_dev, uint32_t stride_floats, uint16_t* density_fp16_dev,
                                       uint32_t n, void* stream);
/* Occupancy march alone (init_rays + advance_pos + generate_next loop with no termination):
 * for each listed pixel writes up to max_samples {t, dt, pos3, mip, cell_idx} records and the count.
 * rec_dev: float[n_pixels*max_samples*5] (t,dt,x,y,z), idx_dev: uint32[n_pixels*max_samples*2] (mip, cell),
 * count_dev: uint32[n_pixels] (total occupied samples on the ray, may exceed max_samples). */
NsbStatus nsb_march_trace(NsbContext* ctx, const NsbFrame* frame, const uint32_t* pixels_dev, uint32_t n_pixels,
                          uint32_t max_samples, float* rec_dev, uint32_t* idx_dev, uint32_t* count_dev, void* stream);

/* ---- per-edit rebuild on the device (SURVEY.md §8f-1) --------------------------------------------------------------
 * What GrowingSelection::update_tet_mesh (growing_selection.cu:1615) does on the host per gizmo drag, for the cage operator at
 * index op_index of the list given to nsb_set_edit_ops, without moving the operator's arrays off the device:
 *   Cage::interpolate_with_mvc (cage.cu:39-55) -> TetMesh::post_update_vertices (tet_mesh.cu:13-20) ->
 *   TetMesh::update_local_rotations (tet_mesh.cu:38-74) -> TetMesh::build_tet_grid (tet_mesh.cu:369-667; upload :651-667). */
/* weights: HOST float [n_vertices x n_cage_vertices] of Cage::compute_mvc (cage.cu:7-36), computed once per cage. */
NsbStatus nsb_cage_attach_mvc(NsbContext* ctx, int32_t op_index, const float* weights, uint32_t n_cage_vertices);
/* cage_vertices: HOST float [n_cage_vertices x 3], the dragged cage. Rewrites the operator's vertices, boxes, rotations (if it
 * was uploaded with local_rotations) and tet lookup table in place. Synchronises the stream once (the list length). */
NsbStatus nsb_cage_deform(NsbContext* ctx, int32_t op_index, const float* cage_vertices, uint32_t n_cage_vertices, void* stream);
/* Reads an operator's current arrays back (any pointer may be NULL): vertices [3*n_vertices], rotations [9*n_tets],
 * lut_offsets [NSB_GRID_CELLS+1], lut_idx [idx_capacity >= *n_idx], boxes [12] = bbox min,max, warped bbox min,max. */
NsbStatus nsb_cage_download(NsbContext* ctx, int32_t op_index, float* vertices, float* rotations, uint32_t* lut_offsets, uint32_t* lut_idx,
                            uint64_t idx_capacity, uint64_t* n_idx, float* boxes);
/* replaces TetMesh::vanish (tet_mesh.cu:251-363, clear_grid :239-248), the cage tool's "Vanish!" button (growing_selection.cu:184-194), for the
 * cage operator op_index of the uploaded list: every cell, at each of the 5 cascades, that one of the operator's CURRENT tets touches
 * (its vertices as nsb_set_edit_ops uploaded them or the last nsb_cage_deform rebuilt them; the cell test of build_tet_grid: a cell corner
 * inside the tet or a tet face hitting the cell box) gets density 0.0f in the context's running density grid and its bit cleared in the
 * context's occupancy bitfield, at its own cascade. The grid mean, the max-pooled coarser cascades, the EMA step and the rng are left as
 * they are, as vanish leaves them. The next nsb_render sees the result.
 * Differences from the reference: a context with a bitfield (nsb_upload_occupancy) but no running density grid has its bitfield
 * cleared only (the reference always has a grid).
 * A later nsb_update_density_grid refills vanished cells from the network: the reference's GUI turns auto-clean off after vanishing
 * for that reason; this library has no auto-clean, so the caller decides when to update. The host's copy of the grid (the reference's
 * m_nerf.density_grid) is stale until nsb_download_density_grid.
 * n_cells_cleared (may be NULL): if given, receives the number of cells whose density or bit changed, and the call synchronises
 * the stream; otherwise it is stream-ordered and does not synchronise. Allocates nothing.
 * Errors: NSB_ERR_INVALID for an index out of range or an operator that is not a cage with tets, NSB_ERR_STATE without occupancy. */
NsbStatus nsb_cage_vanish(NsbContext* ctx, int32_t op_index, uint64_t* n_cells_cleared, void* stream);

/* ---- membrane (Poisson) boundary values (SURVEY.md §8f-4) ------------------------------------------------------------ */
/* The members GrowingSelection::compute_poisson_boundary reads (growing_selection.cu:2220-2348). */
typedef struct {
	uint32_t sampling_width;     /* m_poisson_editing.sh_sampling_width (10): sampling_width^2 directions per point */
	uint32_t hemisphere_width;   /* m_hemisphere_width (10): the divisor of the stratified (u,v) */
	uint64_t seed;               /* the reference jitters with unseeded std::rand(); here: tcnn pcg32 seeded with this value,
	                                two draws (u then v) per sample in (point, i, j) order */
	float    train_aabb_min[3], train_aabb_max[3]; /* m_aabb */
	int32_t  rgb_activation, density_activation;    /* NsbActivation */
	int32_t  is_inside;          /* is_inside: zero the density where the context's occupancy grid is empty (filter_empty :2200-2218) */
} NsbBoundarySampling;
/* replaces GrowingSelection::compute_poisson_boundary: points HOST [n_points x 3] (proxy-cage vertices, world units);
 * density_out HOST [n_points] (density of each point's first sample), shs_out HOST [n_points x 27] (SH9RGB, column-major 9 x 3:
 * the Monte-Carlo projection 4*pi/n * sum project_sh9(dir, rgb), sh_utils.cu:30-70). Directions are generated on the host like
 * the reference does; inference, activation and the projection run on the device. Synchronises. */
NsbStatus nsb_poisson_boundary(NsbContext* ctx, const float* points, uint32_t n_points, const NsbBoundarySampling* params,
                               float* density_out, float* shs_out);
/* replaces GrowingSelection::interpolate_poisson_boundary (growing_selection.cu:2350-2398) for the cage operator op_index: blends
 * the per-cage-vertex inside/outside densities and SHs through gamma_coordinates (HOST [n_vertices x n_cage_vertices], Cage::compute_mvc
 * with gamma) into the operator's boundary_shs / boundary_outside_density / boundary_residual_density arrays on the device, and sets
 * residual_amplitude / apply_poisson. boundary_*_out (HOST, may be NULL) receive the arrays ([27*n_vertices], [n_vertices] x 2). */
NsbStatus nsb_cage_set_membrane(NsbContext* ctx, int32_t op_index, const float* gamma_coordinates, uint32_t n_cage_vertices,
                                const float* inside_density, const float* outside_density, const float* inside_shs, const float* outside_shs,
                                float residual_amplitude, int32_t apply_poisson,
                                float* boundary_shs_out, float* boundary_outside_density_out, float* boundary_residual_density_out);

/* ---- host-side geometry (the per-edit level; reference runs these on the CPU too) -------- */
/* replaces TetMesh::build_tet_grid (tet_mesh.cu:369-667): CSR tet lookup over 5x128^3 cells for the
 * given vertex set. offsets: [NSB_GRID_CELLS+1]; idx: caller buffer of capacity idx_capacity; *n_idx = needed.
 * bitfield (may be NULL): [NSB_BITFIELD_BYTES], set where a tet touches the cell. */
NsbStatus nsb_build_tet_grid(const float* vertices, uint32_t n_vertices, const uint32_t* tets, uint32_t n_tets,
                             uint32_t* offsets, uint32_t* idx, uint64_t idx_capacity, uint64_t* n_idx, uint8_t* bitfield);
/* replaces Cage::compute_mvc (cage.cu:7-36, mvc.h:126-188): weights [n_points x n_cage_vertices]. */
NsbStatus nsb_compute_mvc(const float* cage_vertices, uint32_t n_cage_vertices, const uint32_t* cage_triangles, uint32_t n_triangles,
                          const float* points, uint32_t n_points, float gamma, float* weights);
/* replaces Cage::interpolate_with_mvc (cage.cu:39-55). */
NsbStatus nsb_interpolate_with_mvc(const float* weights, uint32_t n_points, uint32_t n_cage_vertices,
                                   const float* cage_vertices, float* points_out);
/* replaces TetMesh::update_local_rotations (tet_mesh.cu:38-74): rotations [9*n_tets] column-major. */
NsbStatus nsb_local_rotations(const float* vertices, const float* original_vertices, const uint32_t* tets, uint32_t n_tets, float* rotations);

/* ---- mesh extraction (ABI 4): Testbed::marching_cubes (testbed_nerf.cu:4614-4649), as the GUI's "Mesh it!" (testbed.cu:932-942),
 * compute_marching_cubes_mesh (python_api.cu:105-126) and compute_and_save_marching_cubes_mesh (testbed.cu:337-343) run it ---------- */
typedef struct {
	int32_t res[3];                               /* grid points per axis: positive multiples of 16 (testbed_nerf.cu:4615-4617) */
	float   aabb_min[3], aabb_max[3];             /* the box sampled (m_render_aabb by default) */
	float   train_aabb_min[3], train_aabb_max[3]; /* m_aabb */
} NsbGridQuery;
/* replaces Testbed::get_density_on_grid (testbed_nerf.cu:4538-4586) in NeRF mode: density_dev (DEVICE float[res_x*res_y*res_z], x fastest)
 * receives float(raw fp16 density output) at aabb_min + (x/res_x, y/res_y, z/res_z) * (aabb_max - aabb_min), or -10000 where the context's
 * running density grid (Testbed::Nerf::density_grid) is below NERF_MIN_OPTICAL_THICKNESS at that position (grid_samples_half_to_float :465-481).
 * NSB_ERR_STATE without a model or a density grid. Stream-ordered. */
NsbStatus nsb_density_on_grid(NsbContext* ctx, const NsbGridQuery* query, float* density_dev, void* stream);
/* replaces marching_cubes_gpu (marching_cubes.cu:730-758) on any DEVICE float grid (x fastest; e.g. the output above, or
 * GrowingSelection::extract_fine_mesh's 0/1 selection grid, growing_selection.cu:2096-2162): builds the mesh into arrays the context owns.
 * Vertices are the reference's edge crossings bit for bit (gen_vertices :217-265), ordered by (grid point, axis x, y, z); triangles by
 * (cell, table order) with the table of nsb_mc_table.h, so two calls give the same arrays. *n_vertices, *n_indices: exact counts.
 * Synchronises the stream once, for the counts. Scratch: 4 B per grid point. */
NsbStatus nsb_marching_cubes(NsbContext* ctx, const float* density_dev, const int32_t res[3], const float aabb_min[3], const float aabb_max[3], float thresh,
                             uint64_t* n_vertices, uint64_t* n_indices, void* stream);
/* replaces compute_mesh_1ring's normals (marching_cubes.cu:656-662, accumulate_1ring :267-302) and Testbed::compute_mesh_vertex_colors
 * (testbed_nerf.cu:4515-4536) for the last nsb_marching_cubes mesh: normal = sum of (pb-pa)x(pa-pc) over the vertex's triangles in
 * triangle order (not normalised, like m_mesh.vert_normals); colour = the network at the vertex, direction normalize(pos - 0.5),
 * through network_to_rgb and, when linear_colors, linear_to_srgb (extract_srgb_with_activation :338-351). Stream-ordered. */
NsbStatus nsb_mesh_shade(NsbContext* ctx, const float train_aabb_min[3], const float train_aabb_max[3], int32_t rgb_activation, int32_t linear_colors, void* stream);
/* Copies the mesh back (HOST pointers, any may be NULL; synchronises the device). vertices / normals / colors: [3 * vertex_rows];
 * vertex_rows may be up to n_vertices rounded up to 128, the reference's row count (marching_cubes.cu:751-753): the padding rows are
 * at the origin with a zero normal and the network's colour there. indices: [index_capacity >= n_indices]. */
NsbStatus nsb_mesh_download(NsbContext* ctx, float* vertices, float* normals, float* colors, uint64_t vertex_rows, uint32_t* indices,
                            uint64_t index_capacity);

/* ---- mesh optimisation (ABI 5): Testbed::optimise_mesh_step (testbed_nerf.cu:4470-4513), the GUI's "Optimize mesh" (testbed.cu:992-995,
 * 1759-1761) ---------------------------------------------------------------------------------------------------------------------------- */
/* replaces NerfNetwork::input_gradient(stream, 3, ...) together with NerfNetwork::density: the gradient of the raw density output with
 * respect to the warped position (not rescaled to world units), through the density MLP and the hash grid, under the context's accumulator
 * policy. coords_dev: n NerfCoordinate rows as for nsb_density. grad_dev: the 3 position floats of row i at grad_dev + i * grad_stride_floats
 * (nothing else is written; grad_dev == coords_dev with stride 7 is allowed, as the reference calls it in place). density_fp16_dev (may be
 * NULL): fp16 [n_padded], the raw density = row 0 of nsb_density's output. dfeat_fp16_dev (may be NULL): fp16 [32 x n_padded] row-major,
 * dL/d(grid features) scaled by 128 (tcnn's backprop_scale). NSB_ERR_STATE without a model. Stream-ordered. */
NsbStatus nsb_density_gradient(NsbContext* ctx, const float* coords_dev, uint32_t n, float* grad_dev, uint32_t grad_stride_floats, uint16_t* density_fp16_dev,
                               uint16_t* dfeat_fp16_dev, uint32_t n_padded, void* stream);
/* The members of Testbed::m_mesh that optimise_mesh_step reads (testbed.h; defaults marching_cubes.h:32-34: 2048, 128, 1). */
typedef struct {
	float thresh;                                 /* m_mesh.thresh: the iso-value the vertices are pushed towards */
	float smooth_amount, density_amount, inflate_amount;
	float train_aabb_min[3], train_aabb_max[3];   /* m_aabb */
} NsbMeshOptimise;
/* replaces Testbed::optimise_mesh_step(n_steps) on the context's mesh: per step, the density and its position gradient at every vertex row
 * (the padding rows included), the 1-ring centroid and area-weighted normal of each vertex (summed in triangle order), the opt gradient
 * normalize(grad) * sign(density - thresh) * density_amount + (v - centroid) * smooth_amount - normalize(normal) * inflate_amount, and one
 * Adam step (tcnn, learning rate 1e-4, beta1 0.9, beta2 0.99, epsilon 1e-8; every coordinate a non-matrix parameter with its own step
 * counter, skipped while its gradient is 0). The indices do not change and the colours are not recomputed; the normals left behind are those
 * of the positions before the last step. Adam state (48 B per vertex row) is allocated on the first call and restarts with the first call
 * after each nsb_marching_cubes. NSB_ERR_STATE without a model or a mesh. Stream-ordered. */
NsbStatus nsb_mesh_optimise(NsbContext* ctx, const NsbMeshOptimise* params, uint32_t n_steps, void* stream);

/* ---- density and RGBA slices (ABI 6): the export panel's "Save density PNG" (Testbed::compute_and_save_png_slices, testbed.cu:345-366,
 * python_api.cu:458) and "Save RGBA PNG sequence" (testbed.cu:956-966). The caller writes the PNG files from the pixels; none of these
 * calls allocates in the context ------------------------------------------------------------------------------------------------------ */
/* replaces Testbed::get_rgba_on_grid (testbed_nerf.cu:4588-4612): rgba_dev (DEVICE float4[res_x*res_y*res_z], x fastest, 16-byte aligned)
 * receives, at the grid positions of nsb_density_on_grid over query->aabb (the reference samples m_render_aabb) seen from direction ray_dir,
 * compute_nerf_density (:624-635) of the full network's output: a = clamp(1 - exp(-network_to_density(density) / 100), 0, 1) and
 * rgb = network_to_rgb(rgb) * a, in one pass without the reference's position buffer (28 B per point) or its 1M-point batches. Same res rules
 * as nsb_density_on_grid; no density grid is needed (the reference applies no filter here). NSB_ERR_STATE without a model. Stream-ordered. */
NsbStatus nsb_rgba_on_grid(NsbContext* ctx, const NsbGridQuery* query, const float ray_dir[3], int32_t rgb_activation, int32_t density_activation,
                           float* rgba_dev, void* stream);
/* The size of save_density_grid_to_png's mosaic (marching_cubes.cu:938-945): with res' = (res_x, res_z, res_y) when swap_y_z, else res,
 * ndown = (uint32_t)sqrtf(res'_z), nacross = ceil(res'_z / ndown), *w = res_x * nacross, *h = res'_y * ndown. Needs no GPU. */
NsbStatus nsb_density_png_extent(const int32_t res[3], int32_t swap_y_z, uint32_t* w, uint32_t* h);
/* replaces the host loops of save_density_grid_to_png (marching_cubes.cu:898-974) on a DEVICE float grid (x fastest; any positive res
 * with a 32-bit point count), without copying the grid to the host. pixels_dev: DEVICE uint8[w * h] (nsb_density_png_extent), the
 * bytes the reference hands to stbi_write_png: tile (i, j) shows slice j * nacross + i, pixel (x, y) of it is
 * (uint8_t)clamp((d - thresh) * (128 / density_range) + 128.5, 0, 255) with the product and sum rounded separately, rows flipped in y
 * unless swap_y_z; tiles past the last slice are 0. counts_dev: DEVICE uint64[2], the logged #zero-x voxels (cells with corners on both
 * sides of thresh) and #lattice near zero-x (grid points with a 6-neighbour on the other side), both over the interior grid points
 * 1 <= x, y, z <= res - 2; integer atomics, so they do not depend on the order. density_range > 0. Needs no model. Stream-ordered. */
NsbStatus nsb_density_png(NsbContext* ctx, const float* density_dev, const int32_t res[3], float thresh, float density_range, int32_t swap_y_z,
                          uint8_t* pixels_dev, uint64_t* counts_dev, void* stream);
/* replaces the host loop of save_rgba_grid_to_png_sequence (marching_cubes.cu:979-1015) on a DEVICE float4 grid (e.g. nsb_rgba_on_grid's,
 * 16-byte aligned): pixels_dev (DEVICE, 4-byte aligned) receives res'_z images of res_x * res'_y RGBA pixels back to back, slice z being
 * the reference's file %04d_<w>x<h>.png, each channel (uint8_t)clamp(v * 255, 0, 255); res' and the y flip as nsb_density_png. Needs no
 * model. Stream-ordered. */
NsbStatus nsb_rgba_png(NsbContext* ctx, const float* rgba_dev, const int32_t res[3], int32_t swap_y_z, uint8_t* pixels_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NERFSHOP_B200_H */
