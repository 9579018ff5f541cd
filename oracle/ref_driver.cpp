// ref_driver.cpp — C entry points around the reference's OWN render-path sources, compiled for the CPU (oracle/_ref).
//
// TEST INFRASTRUCTURE ONLY: built by oracle/ref_build.py into oracle/_ref/libnerfshop_ref.so, loaded by tests/ (and nothing
// else) to pin oracle/nerfshop_oracle.cpp to code the reference's authors wrote. What is reference code here:
//   every #include <neural-graphics-primitives/...>, <common_nerf.cu> and every "*.inc" (functions cut out of the reference's
//   translation units at build time, see ref_build.py EXTRACTS) — including Testbed::render_nerf, NerfTracer::trace,
//   init_rays_from_camera, all the kernels they launch, the cage/affine kernels, MVC, the 3x3 SVD, TetMesh::build_tet_grid.
// What is ours: this file (argument marshalling from the C-ABI PODs of include/nerfshop_b200.h, the declarations of the
// Testbed members that render_nerf reads, NerfNetwork as a call-back) and oracle/ref_shim/ (stand-ins for the absent
// submodules). tiny-cuda-nn's network is NOT here: NerfNetwork::inference_mixed_precision calls the function pointer the test
// supplies (the oracle's encode + MLPs), so rows a7-a9 stay pinned only by the restatement of the published algorithm.
#include <tiny-cuda-nn/common.h>
#include <tiny-cuda-nn/gpu_matrix.h>
#include <tiny-cuda-nn/gpu_memory.h>
#include <tiny-cuda-nn/random.h>

thread_local uint3_ threadIdx, blockIdx;
thread_local dim3 blockDim, gridDim;
namespace tcnn { bool g_parallel_launch = true; }

#define __CUDACC_EXTENDED_LAMBDA__ 1
#include <functional>
#include <future>
#include <memory>
#include <queue>
#include <thread>
#include <tuple>

#include <neural-graphics-primitives/common.h>
#include <neural-graphics-primitives/common_gl.h>  // oracle/ref_shim shadow: GLuint typedefs only
#include <neural-graphics-primitives/common_device.cuh>
#include <neural-graphics-primitives/common_nerf.h>
#include <neural-graphics-primitives/envmap.cuh>
#include <neural-graphics-primitives/random_val.cuh>
#include <neural-graphics-primitives/editing/edit_operator.h>
#include <neural-graphics-primitives/editing/tools/affine_bounding_box.cuh>
#include <neural-graphics-primitives/editing/tools/selection_utils.h>
#include <neural-graphics-primitives/editing/tools/mvc.h>
#include <neural-graphics-primitives/editing/tools/svd3.h>
#include <neural-graphics-primitives/editing/datastructures/tet_mesh.h>
#include <neural-graphics-primitives/editing/datastructures/cage.h>

#include <common_nerf.cu>  // /root/reference/src/common_nerf.cu, whole file

#include "../include/nerfshop_b200.h"

static std::shared_ptr<void> nsb_ref_alloc(size_t bytes) { return std::shared_ptr<void>(calloc(bytes, 1), free); }
#include "ref_common.inl"


using namespace ngp;

static Eigen::Matrix<float, 3, 4> cam34(const float* m) { Eigen::Matrix<float, 3, 4> r; memcpy(r.data(), m, 12 * sizeof(float)); return r; }

// launches kernel for the single linear index i (threadIdx.x + blockIdx.x * blockDim.x == i)
static inline void set_linear_thread(uint32_t i) { blockDim = dim3(1); gridDim = dim3(1); blockIdx = {i, 0, 0}; threadIdx = {0, 0, 0}; }

extern "C" {

int ref_set_parallel(int on) { tcnn::g_parallel_launch = on != 0; return 0; }

// ---- scalar functions, vectorised over n (random_val.cuh, common_nerf.cu, bounding_box.cuh, common_device.cuh) --------
void ref_ld_random_val(uint32_t n, const uint32_t* index, const uint32_t* seed, float* out) { for (uint32_t i = 0; i < n; ++i) out[i] = ld_random_val(index[i], seed[i]); }
void ref_ld_random_pixel_offset(uint32_t spp, float* out) { Eigen::Vector2f o = ld_random_pixel_offset(spp); out[0] = o.x(); out[1] = o.y(); }
void ref_morton3D(uint32_t n, const uint32_t* xyz, uint32_t* out) { for (uint32_t i = 0; i < n; ++i) out[i] = tcnn::morton3D(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]); }
void ref_mip(uint32_t n, const float* pos, const float* dt, int* mip_pos, int* mip_dt, uint32_t* cell /*at mip_dt*/) {
	for (uint32_t i = 0; i < n; ++i) {
		Eigen::Vector3f p(pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]);
		mip_pos[i] = mip_from_pos(p);
		mip_dt[i] = mip_from_dt(dt[i], p);
		cell[i] = cascaded_grid_idx_at(p, (uint32_t)mip_dt[i]);
	}
}
void ref_calc_dt(uint32_t n, const float* t, float cone, float* out) { for (uint32_t i = 0; i < n; ++i) out[i] = calc_dt(t[i], cone); }
void ref_advance_to_next_voxel(uint32_t n, const float* t, float cone, const float* pos, const float* dir, const uint32_t* res, float* out) {
	for (uint32_t i = 0; i < n; ++i) {
		Eigen::Vector3f p(pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]), d(dir[3 * i], dir[3 * i + 1], dir[3 * i + 2]);
		out[i] = advance_to_next_voxel(t[i], cone, p, d, d.cwiseInverse(), res[i]);
	}
}
void ref_warp(uint32_t n, const float* pos, const float* dir, const float* dt, const float* amin, const float* amax, float* out /*7 per: wp, wdt, wd*/, float* back /*7 per: unwarp of out*/) {
	BoundingBox aabb = bb(amin, amax);
	for (uint32_t i = 0; i < n; ++i) {
		Eigen::Vector3f p(pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]), d(dir[3 * i], dir[3 * i + 1], dir[3 * i + 2]);
		Eigen::Vector3f wp = warp_position(p, aabb), wd = warp_direction(d);
		float wdt = warp_dt(dt[i]);
		float* o = out + 7 * (size_t)i;
		o[0] = wp.x(); o[1] = wp.y(); o[2] = wp.z(); o[3] = wdt; o[4] = wd.x(); o[5] = wd.y(); o[6] = wd.z();
		Eigen::Vector3f up = unwarp_position(wp, aabb), ud = unwarp_direction(wd);
		float* b = back + 7 * (size_t)i;
		b[0] = up.x(); b[1] = up.y(); b[2] = up.z(); b[3] = unwarp_dt(wdt); b[4] = ud.x(); b[5] = ud.y(); b[6] = ud.z();
	}
}
void ref_ray_intersect(uint32_t n, const float* o, const float* d, const float* mn, const float* mx, float* tmin_out, uint8_t* contains_out) {
	BoundingBox box = bb(mn, mx);
	for (uint32_t i = 0; i < n; ++i) {
		Eigen::Vector3f oo(o[3 * i], o[3 * i + 1], o[3 * i + 2]), dd(d[3 * i], d[3 * i + 1], d[3 * i + 2]);
		tmin_out[i] = box.ray_intersect(oo, dd).x();
		contains_out[i] = box.contains(oo) ? 1 : 0;
	}
}
void ref_srgb_to_linear(uint32_t n, const float* in, float* out) { for (uint32_t i = 0; i < n; ++i) out[i] = srgb_to_linear(in[i]); }
void ref_evaluate_sh9(uint32_t n, const float* sh /*27 per*/, const float* dir, float* out) {
	for (uint32_t i = 0; i < n; ++i) {
		SH9RGB s; memcpy(s.data(), sh + 27 * (size_t)i, 27 * sizeof(float));
		Eigen::Vector3f r = evaluate_sh9(s, Eigen::Vector3f(dir[3 * i], dir[3 * i + 1], dir[3 * i + 2]));
		out[3 * i] = r.x(); out[3 * i + 1] = r.y(); out[3 * i + 2] = r.z();
	}
}
void ref_activations(uint32_t n, const float* in, int act, float* rgb_out, float* density_out) {
	for (uint32_t i = 0; i < n; ++i) { rgb_out[i] = network_to_rgb(in[i], (ENerfActivation)act); density_out[i] = network_to_density(in[i], (ENerfActivation)act); }
}
void ref_pcg32(uint64_t initstate, uint64_t initseq, uint64_t advance, uint32_t n, uint32_t* out_uint, float* out_float) {
	default_rng_t rng(initstate, initseq);
	if (advance) rng.advance((int64_t)advance);
	default_rng_t r2 = rng;
	for (uint32_t i = 0; i < n; ++i) out_uint[i] = rng.next_uint();
	for (uint32_t i = 0; i < n; ++i) out_float[i] = r2.next_float();
}
// generate_grid_samples_nerf_nonuniform (common_nerf.cu:179-208): the occupancy update's sample draw
void ref_grid_samples(uint32_t n, uint64_t rng_state, uint64_t rng_inc, uint32_t step, const float* amin, const float* amax, const float* grid_in, uint32_t n_cascades, float thresh,
                      float* out_pos /*3 per, warped*/, uint32_t* out_idx) {
	default_rng_t rng; rng.state = rng_state; rng.inc = rng_inc;
	std::vector<NerfPosition> pos(n, NerfPosition(Eigen::Vector3f::Zero(), 0.f));
	tcnn::linear_kernel(generate_grid_samples_nerf_nonuniform, 0, nullptr, n, rng, step, bb(amin, amax), grid_in, pos.data(), out_idx, n_cascades, thresh);
	for (uint32_t i = 0; i < n; ++i) { out_pos[3 * i] = pos[i].p.x(); out_pos[3 * i + 1] = pos[i].p.y(); out_pos[3 * i + 2] = pos[i].p.z(); }
}

// Testbed::update_density_grid_mean_and_bitfield (testbed_nerf.cu:3642-3658) after its reduce_sum: grid_to_bitfield over all cascades with the given
// mean, then bitfield_max_pool level by level. grid: float[5*128^3]; bits: uint8[5*128^3/8].
void ref_grid_to_bitfield(const float* grid, float mean, uint8_t* bits) {
	const uint32_t n_elements = NERF_GRIDSIZE() * NERF_GRIDSIZE() * NERF_GRIDSIZE();
	memset(bits, 0, grid_mip_offset(NERF_CASCADES()) / 8);
	tcnn::linear_kernel(grid_to_bitfield, 0, nullptr, n_elements / 8 * NERF_CASCADES(), grid, bits, &mean);
	for (uint32_t level = 1; level < NERF_CASCADES(); ++level)
		tcnn::linear_kernel(bitfield_max_pool, 0, nullptr, n_elements / 64, bits + grid_mip_offset(level - 1) / 8, bits + grid_mip_offset(level) / 8);
}

// ---- ray generation + occupancy march with the reference's kernels, one sample per call of generate_next (n_steps = 1) ----
// For every listed pixel: init_rays_with_payload_kernel_nerf -> advance_pos_nerf -> generate_next_nerf_network_inputs x max_samples.
// rec: per pixel per sample 8 floats = the NerfCoordinate the reference would feed the network (warped pos 3, warped dt, warped dir 3)
// + payload.t after the step; ray: per pixel 8 floats = origin 3, dir 3, t after init_rays (ray start), t after advance_pos (first sample)
int ref_march_trace(const NsbFrame* f, const uint8_t* bitfield, const uint32_t* pixels, uint32_t n_pixels, uint32_t max_samples, float* rec, float* ray, uint32_t* count, uint8_t* alive_after_init) {
	const uint32_t W = (uint32_t)f->width, H = (uint32_t)f->height, N = W * H;
	std::vector<NerfPayload> payloads(N);
	std::vector<Array4f> fb(N, Array4f::Zero());
	std::vector<float> depth(N, 0.f);
	std::vector<NerfCoordinate> input((size_t)N, NerfCoordinate(Vector3f::Zero(), Vector3f::Zero(), 0.f));
	const BoundingBox render_aabb = bb(f->render_aabb_min, f->render_aabb_max), train_aabb = bb(f->train_aabb_min, f->train_aabb_max);
	const Eigen::Matrix<float, 3, 4> c0 = cam34(f->camera0), c1 = cam34(f->camera1);
	const Vector2f focal(f->focal_length[0], f->focal_length[1]);
	const Vector4f rs(f->rolling_shutter[0], f->rolling_shutter[1], f->rolling_shutter[2], f->rolling_shutter[3]);
#pragma omp parallel for schedule(dynamic, 16)
	for (uint32_t k = 0; k < n_pixels; ++k) {
		const uint32_t pix = pixels[k], x = pix % W, y = pix / W;
		blockDim = dim3(1, 1, 1); gridDim = dim3(W, H, 1); blockIdx = {x, y, 0}; threadIdx = {0, 0, 0};
		init_rays_with_payload_kernel_nerf(f->spp_index, payloads.data(), Vector2i((int)W, (int)H), focal, c0, c1, rs, Vector2f(f->screen_center[0], f->screen_center[1]),
		                                   (bool)f->snap_to_pixel_centers, render_aabb, f->focus_z > 0.f ? f->focus_z : 1.0f /*plane_z = m_slice_plane_z + m_scale*/, f->dof, frame_camera_distortion(f), nullptr, Vector2i::Zero(),
		                                   fb.data(), depth.data(), f->distortion_dev, Vector2i(f->distortion_resolution[0], f->distortion_resolution[1]), (ERenderMode)f->render_mode);
		NerfPayload& p = payloads[pix];
		float* rr = ray + 8 * (size_t)k;
		rr[0] = p.origin.x(); rr[1] = p.origin.y(); rr[2] = p.origin.z(); rr[3] = p.dir.x(); rr[4] = p.dir.y(); rr[5] = p.dir.z(); rr[6] = p.t;
		alive_after_init[k] = p.alive ? 1 : 0;
		set_linear_thread(pix);
		advance_pos_nerf(N, render_aabb, c1.col(2), focal, f->spp_index, payloads.data(), bitfield, (uint32_t)f->min_mip, f->cone_angle_constant);
		rr[7] = p.t;
		uint32_t c = 0;
		while (p.alive && c < max_samples) {
			set_linear_thread(pix);
			generate_next_nerf_network_inputs(N, render_aabb, train_aabb, focal, c1.col(2), payloads.data(), PitchedPtr<NerfCoordinate>(input.data(), 1, 0, 0), 1, bitfield,
			                                  (uint32_t)f->min_mip, f->cone_angle_constant, Vector3f::Zero());
			if (p.n_steps == 0) break;  // left the render aabb
			const NerfCoordinate& nc = input[pix];
			float* o = rec + ((size_t)k * max_samples + c) * 8;
			o[0] = nc.pos.p.x(); o[1] = nc.pos.p.y(); o[2] = nc.pos.p.z(); o[3] = nc.dt; o[4] = nc.dir.d.x(); o[5] = nc.dir.d.y(); o[6] = nc.dir.d.z(); o[7] = p.t;
			++c;
		}
		count[k] = c;
	}
	return 0;
}

// ---- Testbed::render_nerf, the reference's own, end to end; the network is the call-back ------------------------------------
// fb / depth: float4[W*H] / float[W*H], zero-initialised by the caller like CudaRenderBuffer::clear_frame_buffer.
int ref_render(const NsbFrame* f, const uint8_t* bitfield, const NsbEditOp* ops, int n_ops, ref_inference_fn fn, void* user, float* fb, float* depth, uint64_t* stats /*4: n_hit, n_inferred, n_calls, n_rays*/) {
	try {
		Testbed tb;
		tb.m_render_mode = (ERenderMode)f->render_mode;
		tb.m_snap_to_pixel_centers = f->snap_to_pixel_centers != 0;
		tb.m_render_aabb = bb(f->render_aabb_min, f->render_aabb_max);
		tb.m_aabb = bb(f->train_aabb_min, f->train_aabb_max);
		tb.m_nerf.density_grid_bitfield.copy_from_host(bitfield, NSB_BITFIELD_BYTES);
		tb.m_nerf.show_accel = f->show_accel ? f->min_mip : -1;  // the reference derives min_mip from show_accel; without the override min_mip is 0
		tb.m_nerf.cone_angle_constant = f->cone_angle_constant;
		tb.m_nerf.training.dataset.scale = 1.0f / f->depth_scale;
		tb.m_nerf.training.linear_colors = f->linear_colors != 0;
		tb.m_nerf.rgb_activation = (ENerfActivation)f->rgb_activation;
		tb.m_nerf.density_activation = (ENerfActivation)f->density_activation;
		tb.m_nerf.rendering_min_transmittance = f->min_transmittance;
		tb.m_nerf.tracer.m_poisson_target = f->poisson_target != 0;
		set_frame_extras(tb, f);
		for (int i = 0; i < n_ops; ++i) tb.m_nerf.tracer.add_edit_operator(make_op(ops[i]));
		NerfNetwork<network_precision_t> net; net.fn = fn; net.user = user;
		CudaRenderBuffer rb; rb.res = Vector2i(f->width, f->height); rb.m_spp = f->spp_index; rb.fb = (Array4f*)fb; rb.depth = depth;
		tb.render_nerf(net, rb, rb.res, Vector2f(f->focal_length[0], f->focal_length[1]), cam34(f->camera0), cam34(f->camera1),
		               Vector4f(f->rolling_shutter[0], f->rolling_shutter[1], f->rolling_shutter[2], f->rolling_shutter[3]), Vector2f(f->screen_center[0], f->screen_center[1]),
		               f->apply_operators != 0, nullptr);
		if (stats) { stats[0] = 0; stats[1] = net.n_inferred; stats[2] = net.n_calls; stats[3] = (uint64_t)f->width * f->height; }
		return 0;
	} catch (const std::exception& e) {
		fprintf(stderr, "ref_render: %s\n", e.what());
		return 1;
	}
}

// ---- Testbed::update_density_grid_nerf_operator + update_density_grid_mean_and_bitfield, the reference's own (testbed_nerf.cu:3533-3658) ----
// grid: float[5*128^3] in/out (the running density grid), bits: uint8[5*128^3/8] out, mean_out: density_grid_mean. NerfNetwork::density is the call-back.
int ref_update_density_grid(const NsbGridUpdate* u, const NsbEditOp* ops, int n_ops, ref_density_fn dfn, void* user, float* grid, uint8_t* bits, float* mean_out) {
	try {
		const uint32_t n_cells = NERF_GRIDSIZE() * NERF_GRIDSIZE() * NERF_GRIDSIZE() * NERF_CASCADES();
		Testbed tb;
		tb.m_aabb = bb(u->train_aabb_min, u->train_aabb_max);
		tb.m_nerf.density_grid.resize(n_cells);
		tb.m_nerf.density_grid.copy_from_host(grid, n_cells);
		tb.m_nerf.density_grid_ema_step = u->ema_step;
		tb.m_nerf.max_cascade = (uint32_t)u->n_cascades - 1;
		tb.m_nerf.training.density_grid_decay = u->decay;
		tb.m_nerf.density_activation = (ENerfActivation)u->density_activation;
		tb.m_rng.state = u->rng_state; tb.m_rng.inc = u->rng_inc;
		if (u->apply_operators) for (int i = 0; i < n_ops; ++i) tb.m_nerf.tracer.add_edit_operator(make_op(ops[i]));
		tb.m_nerf_network = std::make_shared<NerfNetwork<network_precision_t>>();
		tb.m_nerf_network->dfn = dfn; tb.m_nerf_network->user = user;
		tcnn::g_scratch_floor = (size_t)n_cells * 12;  // see ref_common.inl: room for the reference's over-long compute_poisson_residual_density launch
		tb.update_density_grid_nerf_operator(u->n_uniform_samples, u->n_nonuniform_samples, u->reset_grid != 0, nullptr);
		tcnn::g_scratch_floor = 0;
		tb.m_nerf.density_grid.copy_to_host(grid, n_cells);
		tb.m_nerf.density_grid_bitfield.copy_to_host(bits, NSB_BITFIELD_BYTES);
		if (mean_out) tb.m_nerf.density_grid_mean.copy_to_host(mean_out, 1);
		return 0;
	} catch (const std::exception& e) {
		fprintf(stderr, "ref_update_density_grid: %s\n", e.what());
		return 1;
	}
}

// ---- accumulate_kernel / tonemap_kernel (render_buffer.cu:217-252, 254-332, 471-501), the reference's own ----
// frame, acc, out: float4[W*H]; background: 4 floats (sRGB); enums = common.h's EColorSpace / ETonemapCurve
int ref_accumulate(int W, int H, const float* frame, float* acc, float sample_count, int color_space) {
#pragma omp parallel for schedule(static)
	for (int y = 0; y < H; ++y)
		for (int x = 0; x < W; ++x) {
			blockDim = dim3(1, 1, 1); gridDim = dim3(W, H, 1); blockIdx = {(uint32_t)x, (uint32_t)y, 0}; threadIdx = {0, 0, 0};
			accumulate_kernel(Vector2i(W, H), (Array4f*)frame, (Array4f*)acc, sample_count, (EColorSpace)color_space);
		}
	return 0;
}
int ref_tonemap(int W, int H, float exposure, const float* background, const float* acc, int color_space, int output_color_space, int curve, int clamp_output, float* out) {
	const Array4f bg(background[0], background[1], background[2], background[3]);
#pragma omp parallel for schedule(static)
	for (int y = 0; y < H; ++y)
		for (int x = 0; x < W; ++x) {
			blockDim = dim3(1, 1, 1); gridDim = dim3(W, H, 1); blockIdx = {(uint32_t)x, (uint32_t)y, 0}; threadIdx = {0, 0, 0};
			tonemap_kernel(Vector2i(W, H), exposure, bg, (Array4f*)acc, (EColorSpace)color_space, (EColorSpace)output_color_space, (ETonemapCurve)curve, clamp_output != 0, 0, (Vector4f*)out);
		}
	return 0;
}

// ---- the membrane blend: the loop of GrowingSelection::interpolate_poisson_boundary (growing_selection.cu:2363-2392), cut out of the member ----
// gamma: [n_tet_vertices][n_cage_vertices]; *_shs: 27 floats per cage vertex; outputs per tet vertex
int ref_membrane_blend(const float* gamma, uint32_t n_tv, uint32_t n_cv, const float* inside_density, const float* outside_density, const float* inside_shs,
                       const float* outside_shs, float* b_shs, float* b_od, float* b_rd) {
	struct Resizable { void resize(size_t) {} };
	struct Mesh {
		std::vector<Eigen::Vector3f> vertices;
		std::vector<std::vector<float>> gamma_coordinates;
		Resizable boundary_shs_gpu, boundary_residual_density_gpu, boundary_outside_density_gpu;
	} mesh, *tet_interpolation_mesh = &mesh;
	struct ProxyCage {
		std::vector<Eigen::Vector3f> vertices;
		std::vector<float> inside_density, outside_density;
		std::vector<SH9RGB> inside_shs, outside_shs;
	} proxy_cage;
	mesh.vertices.resize(n_tv);
	mesh.gamma_coordinates.assign(n_tv, std::vector<float>(n_cv));
	for (uint32_t i = 0; i < n_tv; ++i) for (uint32_t j = 0; j < n_cv; ++j) mesh.gamma_coordinates[i][j] = gamma[(size_t)i * n_cv + j];
	proxy_cage.vertices.resize(n_cv);
	proxy_cage.inside_density.assign(inside_density, inside_density + n_cv);
	proxy_cage.outside_density.assign(outside_density, outside_density + n_cv);
	proxy_cage.inside_shs.resize(n_cv); proxy_cage.outside_shs.resize(n_cv);
	memcpy((void*)proxy_cage.inside_shs.data(), inside_shs, (size_t)n_cv * 27 * sizeof(float));
	memcpy((void*)proxy_cage.outside_shs.data(), outside_shs, (size_t)n_cv * 27 * sizeof(float));
#include "growing_selection.inc"
	}  // closes the cut-out's `for (int i = 0; i < n_tet_vertices; i++) {`
	memcpy(b_shs, boundary_shs_host.data(), (size_t)n_tv * 27 * sizeof(float));
	memcpy(b_od, boundary_outside_density_host.data(), (size_t)n_tv * sizeof(float));
	memcpy(b_rd, boundary_residual_density_host.data(), (size_t)n_tv * sizeof(float));
	return 0;
}

// ---- GrowingSelection::compute_poisson_boundary, the reference's own (growing_selection.cu:2220-2348); its jitter comes from std::rand() ----
// points: [n x 3] world units (proxy-cage vertices); density_out [n], shs_out [n x 27]. The network is the call-back; it sees the sample coordinates.
int ref_poisson_boundary(const float* points, uint32_t n_points, const NsbBoundarySampling* p, const uint8_t* bitfield, ref_inference_fn fn, void* user, float* density_out, float* shs_out) {
	try {
		GrowingSelection gs;
		std::vector<Eigen::Vector3f> pts(n_points);
		for (uint32_t i = 0; i < n_points; ++i) pts[i] = Eigen::Vector3f(points[3 * i], points[3 * i + 1], points[3 * i + 2]);
		gs.proxy_cage.vertices = pts;
		gs.proxy_cage.original_vertices = pts;
		gs.m_poisson_editing.sh_sampling_width = p->sampling_width;
		gs.m_hemisphere_width = p->hemisphere_width;
		gs.m_aabb = bb(p->train_aabb_min, p->train_aabb_max);
		gs.m_rgb_activation = (ENerfActivation)p->rgb_activation;
		gs.m_density_activation = (ENerfActivation)p->density_activation;
		gs.m_density_grid_bitfield.copy_from_host(bitfield, NSB_BITFIELD_BYTES);
		gs.m_nerf_network = std::make_shared<NerfNetwork<network_precision_t>>();
		gs.m_nerf_network->fn = fn; gs.m_nerf_network->user = user;
		gs.compute_poisson_boundary(p->is_inside != 0);
		const std::vector<float>& d = p->is_inside ? gs.proxy_cage.inside_density : gs.proxy_cage.outside_density;
		const std::vector<SH9RGB>& sh = p->is_inside ? gs.proxy_cage.inside_shs : gs.proxy_cage.outside_shs;
		for (uint32_t i = 0; i < n_points; ++i) { density_out[i] = d[i]; memcpy(shs_out + 27 * (size_t)i, sh[i].data(), 27 * sizeof(float)); }
		return 0;
	} catch (const std::exception& e) {
		fprintf(stderr, "ref_poisson_boundary: %s\n", e.what());
		return 1;
	}
}

// ---- EditOperator::map_rays / compute_poisson_full_residuals on a flat batch (reverse list order, testbed_nerf.cu:2868,2899) ----
int ref_map_rays(const NsbEditOp* ops, int n_ops, float* coords /*7 per sample*/, uint8_t* empty_mask, uint32_t n) {
	static_assert(sizeof(NerfCoordinate) == 7 * sizeof(float), "NerfCoordinate layout");
	GPUMatrix<bool> mask(1, n);
	memset(mask.data(), 0, n);
	PitchedPtr<NerfCoordinate> in((NerfCoordinate*)coords, 1, 0, 0);
	for (int i = n_ops - 1; i >= 0; --i) make_op(ops[i])->map_rays(nullptr, in, mask, n);
	for (uint32_t i = 0; i < n; ++i) empty_mask[i] = mask.data()[i] ? 1 : 0;
	return 0;
}
int ref_poisson_residuals(const NsbEditOp* ops, int n_ops, const float* coords, uint32_t n, float* sh /*27 per*/, float* out_density, float* residual_density) {
	std::vector<NerfPayload> payloads(n);
	for (auto& p : payloads) { p.n_steps = 1; p.alive = true; }
	std::vector<SH9RGB> shs(n, SH9RGB::Zero());
	memset(out_density, 0, n * sizeof(float));
	memset(residual_density, 0, n * sizeof(float));
	PitchedPtr<NerfCoordinate> in((NerfCoordinate*)coords, 1, 0, 0);
	for (int i = n_ops - 1; i >= 0; --i) make_op(ops[i])->compute_poisson_full_residuals(nullptr, n, payloads.data(), in, shs.data(), out_density, residual_density);
	for (uint32_t i = 0; i < n; ++i) memcpy(sh + 27 * (size_t)i, shs[i].data(), 27 * sizeof(float));
	return 0;
}
// ---- EditOperator::map_positions / compute_poisson_residual_density on a flat batch (reverse list order, testbed_nerf.cu:3595-3598, 3612-3620) ----
// positions: warped, `stride` floats apart; empty_mask: in/out (only ever set). density: fp16 bits, in/out.
int ref_map_positions(const NsbEditOp* ops, int n_ops, float* positions, uint32_t stride, uint8_t* empty_mask, uint32_t n) {
	static_assert(sizeof(NerfPosition) == 3 * sizeof(float), "NerfPosition layout");
	GPUMatrix<bool> mask(1, n);
	for (uint32_t i = 0; i < n; ++i) mask.data()[i] = empty_mask[i] != 0;
	PitchedPtr<NerfPosition> in((NerfPosition*)positions, 0, 0, (size_t)stride * sizeof(float));
	for (int i = n_ops - 1; i >= 0; --i) make_op(ops[i])->map_positions(nullptr, in, mask, n);
	for (uint32_t i = 0; i < n; ++i) empty_mask[i] = mask.data()[i] ? 1 : 0;
	return 0;
}
int ref_poisson_residual_density(const NsbEditOp* ops, int n_ops, float* positions, uint32_t stride, uint16_t* density, uint32_t n) {
	static_assert(sizeof(tcnn::network_precision_t) == sizeof(uint16_t), "fp16 density");
	PitchedPtr<NerfPosition> in((NerfPosition*)positions, 0, 0, (size_t)stride * sizeof(float));
	for (int i = n_ops - 1; i >= 0; --i) make_op(ops[i])->compute_poisson_residual_density(nullptr, n, in, (tcnn::network_precision_t*)density);
	return 0;
}

// ---- per-edit geometry: MVC (mvc.h:126-188 through Cage::compute_mvc), Kabsch rotations (tet_mesh.cu:38-74 + svd3.h), LUT build ----
// weights: [n_points x n_cage_vertices] row-major
int ref_compute_mvc(const float* cage_vertices, uint32_t n_cv, const uint32_t* cage_tris, uint32_t n_tris, const float* points, uint32_t n_points, float* weights, float gamma, int original) {
	std::vector<Eigen::Vector3f> cv(n_cv), pts(n_points);
	for (uint32_t i = 0; i < n_cv; ++i) cv[i] = Eigen::Vector3f(cage_vertices[3 * i], cage_vertices[3 * i + 1], cage_vertices[3 * i + 2]);
	for (uint32_t i = 0; i < n_points; ++i) pts[i] = Eigen::Vector3f(points[3 * i], points[3 * i + 1], points[3 * i + 2]);
	std::vector<uint32_t> idx(cage_tris, cage_tris + 3 * (size_t)n_tris);
	Cage<float, Eigen::Vector3f> cage(cv, idx);
	std::vector<std::vector<float>> w;
	std::vector<uint8_t> labels;
	cage.compute_mvc(pts, w, labels, original != 0, gamma);
	for (uint32_t i = 0; i < n_points; ++i) for (uint32_t j = 0; j < n_cv; ++j) weights[(size_t)i * n_cv + j] = w[i][j];
	return 0;
}
struct RefTetMesh {
	std::shared_ptr<TetMesh<float, Eigen::Vector3f>> m;
};
// Builds a TetMesh the way GrowingSelection does (constructor + vertices overwrite + post_update_vertices), then
// update_local_rotations + build_tet_grid. Outputs are copied out of the mesh's (host-backed) GPUMemory members.
int ref_tet_mesh_build(const float* original_vertices, const float* deformed_vertices, uint32_t n_v, const uint32_t* tets, uint32_t n_tets, const float* amin, const float* amax,
                       float* rotations /*9 per tet*/, uint32_t* lut_offsets /*NSB_GRID_CELLS+1*/, uint32_t* lut_idx, uint32_t lut_capacity, uint32_t* n_lut_idx,
                       float* bbox /*12: bbox min,max, warped bbox min,max*/, uint8_t* original_bitfield /*NSB_BITFIELD_BYTES*/) {
	std::vector<Eigen::Vector3f> ov(n_v);
	for (uint32_t i = 0; i < n_v; ++i) ov[i] = Eigen::Vector3f(original_vertices[3 * i], original_vertices[3 * i + 1], original_vertices[3 * i + 2]);
	std::vector<uint32_t> indices, tt(tets, tets + 4 * (size_t)n_tets);
	TetMesh<float, Eigen::Vector3f> mesh(ov, indices, tt, bb(amin, amax));
	for (uint32_t i = 0; i < n_v; ++i) mesh.vertices[i] = Eigen::Vector3f(deformed_vertices[3 * i], deformed_vertices[3 * i + 1], deformed_vertices[3 * i + 2]);
	mesh.post_update_vertices();
	mesh.original_tet_lut_idx.resize(1);  // build_original_tet_grid is not on the render path: skip it (build_tet_grid only checks size() == 0)
	mesh.update_local_rotations(nullptr);
	mesh.build_tet_grid(nullptr);
	for (uint32_t t = 0; t < n_tets; ++t) memcpy(rotations + 9 * (size_t)t, mesh.local_rotations_gpu[t].data(), 9 * sizeof(float));
	memcpy(lut_offsets, mesh.tet_lut_offsets.data(), mesh.tet_lut_offsets.size() * sizeof(uint32_t));
	*n_lut_idx = (uint32_t)mesh.tet_lut_idx.size();
	if (mesh.tet_lut_idx.size() > lut_capacity) return 2;
	memcpy(lut_idx, mesh.tet_lut_idx.data(), mesh.tet_lut_idx.size() * sizeof(uint32_t));
	mesh.original_bitfield_gpu.copy_to_host(original_bitfield, NSB_BITFIELD_BYTES);
	const Eigen::Vector3f v[4] = {mesh.bbox.min, mesh.bbox.max, mesh.warped_bbox.min, mesh.warped_bbox.max};
	for (int k = 0; k < 4; ++k) { bbox[3 * k] = v[k].x(); bbox[3 * k + 1] = v[k].y(); bbox[3 * k + 2] = v[k].z(); }
	return (int)mesh.tet_lut_offsets.size() == (int)NSB_GRID_CELLS + 1 ? 0 : 3;
}
// ---- the edits file's objects through the reference's OWN serialisers (row (f)-3) -----------------------------------------------------------
// kind 0: Cage (cage.h:100-144), 1: TetMesh (tet_mesh.h:137-174), 2: AffineBoundingBox (affine_bounding_box.cuh:116-142, free functions),
// 3: AffineBoundingBox via its to_json() member (:103-114, what AffineDuplication::to_json stores). The JSON text is parsed, read with the
// reference's from_json into its class, written back with its to_json, and returned as text (returns the length needed, or -1 on error).
int ref_json_roundtrip(int kind, const char* text_in, char* text_out, int capacity) {
	try {
		const nlohmann::json in = nlohmann::json::parse(text_in);
		nlohmann::json out;
		if (kind == 0) {
			Cage<float, Eigen::Vector3f> cage;
			from_json(in, cage);
			to_json(out, cage);
		} else if (kind == 1) {
			TetMesh<float, Eigen::Vector3f> mesh;
			from_json(in, mesh);
			to_json(out, mesh);
		} else if (kind == 2 || kind == 3) {
			AffineBoundingBox box;
			from_json(in, box);
			if (kind == 2) to_json(out, box); else out = box.to_json();
		} else {
			return -1;
		}
		const std::string s = out.dump();
		if ((int)s.size() + 1 <= capacity) memcpy(text_out, s.c_str(), s.size() + 1);
		return (int)s.size() + 1;
	} catch (const std::exception& e) {
		fprintf(stderr, "ref_json_roundtrip: %s\n", e.what());
		return -1;
	}
}
void ref_svd3(uint32_t n, const float* A /*9 per, column-major*/, float* R /*U * V^T, column-major*/) {
	for (uint32_t i = 0; i < n; ++i) {
		Eigen::Matrix3f a, U, S, V; memcpy(a.data(), A + 9 * (size_t)i, 9 * sizeof(float));
		svd_eigen(a, U, S, V);
		Eigen::Matrix3f r = U * V.transpose();
		memcpy(R + 9 * (size_t)i, r.data(), 9 * sizeof(float));
	}
}

}  // extern "C"
