// nerfshop_host.hpp — C++ shim over the C ABI (include/nerfshop_b200.h) that keeps the reference's class names and
// member signatures for the render path, so that Testbed::render_frame (src/testbed.cu:2632-2648) can call it the way
// it calls the stock code. Header-only; Eigen-free (cameras are passed as 12 floats, column-major like Eigen's storage).
//
//   ngp_b200::NerfNetwork      <- NerfNetwork<T>            (nerf_network.h:87-120): inference_mixed_precision, density, input_gradient(3)
//   ngp_b200::EditOperator     <- EditOperator              (editing/edit_operator.h:25-94): the POD handed to the tracer + the four device
//                                                            virtuals (map_rays, map_positions, compute_poisson_full_residuals,
//                                                            compute_poisson_residual_density) once the operator is attached to a tracer
//   ngp_b200::NerfTracer       <- Testbed::NerfTracer       (testbed.h:129-240): operator list management, trace == render
//   ngp_b200::render_nerf(...) <- Testbed::render_nerf      (testbed.h:305, testbed_nerf.cu:3066)
//   ngp_b200::get_rgba_on_grid, density_png, rgba_png <- Testbed::get_rgba_on_grid and the pixel loops of save_density_grid_to_png /
//                                                       save_rgba_grid_to_png_sequence (the host keeps its own stbi_write_png)
//   ngp_b200::CameraKeyframe, CameraPath <- CameraKeyframe / CameraPath (camera_path.h:30-97): keyframe arithmetic and the B-spline path in the
//                                           reference's float order (no JSON: the host keeps its own load / save)
//   ngp_b200::render_to_cpu(...)        <- Testbed::render_to_cpu's sub-frame loop (python_api.cu:129-175) and copy back, over
//                                           nsb_render_accumulate; the caller builds the sub-frames (nerfshop_b200/camera_path.py restates how)
//   ngp_b200::reference_image, image_metrics <- scripts/run.py's --test_transforms block (run.py:215-302): read_image and the MSE / SSIM
//                                           of a rendered frame on the device
//
// Errors become std::runtime_error, as CUDA_CHECK_THROW does in the reference (propagates to main.cu:252).
#pragma once

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/nerfshop_b200.h"

// density_png / rgba_png hand host pixels back and need the CUDA runtime for their device scratch; the rest of the shim does not
#if defined(__has_include)
#if __has_include(<cuda_runtime_api.h>)
#include <cuda_runtime_api.h>
#define NSB_HOST_HAVE_CUDART 1
#endif
#endif

namespace ngp_b200 {

inline void check(NsbStatus s, const char* what) {
	if (s != NSB_OK) throw std::runtime_error(std::string(what) + ": " + nsb_last_error());
}

class Context {
public:
	explicit Context(int device = -1) { check(nsb_create(device, &m_ctx), "nsb_create"); }
	~Context() { nsb_destroy(m_ctx); }
	Context(const Context&) = delete;
	Context& operator=(const Context&) = delete;
	NsbContext* get() const { return m_ctx; }

private:
	NsbContext* m_ctx = nullptr;
};

// The network as the render path sees it. `set_params` takes the contiguous fp16 block tcnn::Trainer owns
// ([density MLP][rgb MLP][hash grid], nerf_network_full.h:316-349).
class NerfNetwork {
public:
	NerfNetwork(std::shared_ptr<Context> ctx, const NsbModelDesc& desc) : m_ctx(std::move(ctx)), m_desc(desc) {}
	void set_params(const uint16_t* params_fp16, uint64_t n_params) { check(nsb_upload_model(m_ctx->get(), &m_desc, params_fp16, n_params), "nsb_upload_model"); }
	// the block where tcnn::Trainer keeps it (device memory): no 26 MB round trip through the host
	void set_params_device(const uint16_t* params_fp16_dev, uint64_t n_params) { check(nsb_upload_model_dev(m_ctx->get(), &m_desc, params_fp16_dev, n_params), "nsb_upload_model_dev"); }
	// tcnn's FullyFusedMLP accumulates in __half fragments; NSB_MLP_ACC_F32 (default) accumulates wide (see include/nerfshop_b200.h)
	void set_accumulator(NsbMlpAccumulator policy) { check(nsb_set_mlp_accumulator(m_ctx->get(), policy), "nsb_set_mlp_accumulator"); }
	uint64_t n_params() const { uint64_t n = 0; check(nsb_model_n_params(&m_desc, &n), "nsb_model_n_params"); return n; }
	uint32_t padded_output_width() const { return 16; }          // nerf_network.h: rgb MLP output padded to 16
	uint32_t padded_density_output_width() const { return 16; }
	uint32_t n_extra_dims() const { return 0; }
	// input: 7 x n floats column-major (NerfCoordinate per column), output: fp16 row-major [16 x n_padded] (testbed_nerf.cu:2890-2913)
	void inference_mixed_precision(void* stream, const float* input_dev, uint16_t* output_dev, uint32_t n, uint32_t n_padded) const {
		check(nsb_inference(m_ctx->get(), input_dev, n, output_dev, n_padded, stream), "nsb_inference");
	}
	void density(void* stream, const float* input_dev, uint16_t* output_dev, uint32_t n, uint32_t n_padded) const {
		check(nsb_density(m_ctx->get(), input_dev, n, output_dev, n_padded, stream), "nsb_density");
	}
	// NerfNetwork::input_gradient (nerf_network_full.h:142-221) for the density output (dim 3) only: the gradient w.r.t. the warped
	// position into the first 3 floats of each output row (output_dev == input_dev is allowed, as the reference calls it in place)
	void input_gradient(void* stream, uint32_t dim, const float* input_dev, float* output_dev, uint32_t output_stride_floats, uint32_t n, uint32_t n_padded) const {
		if (dim != 3) throw std::runtime_error("NerfNetwork::input_gradient: only dim 3 (the density) is implemented");
		check(nsb_density_gradient(m_ctx->get(), input_dev, n, output_dev, output_stride_floats, nullptr, nullptr, n_padded, stream), "nsb_density_gradient");
	}

private:
	std::shared_ptr<Context> m_ctx;
	NsbModelDesc m_desc;
};

// An operator is the POD of its kernel arguments; the interactive tooling that produces it (GrowingSelection, TetGen, ...)
// stays in the host application. CageDeformation / AffineDuplication fill the respective half of NsbEditOp. Once added to a
// NerfTracer the operator knows its slot in the uploaded list and the device virtuals of the reference's EditOperator work
// (edit_operator.h:43,45,68,81; PitchedPtr arguments become pointer + stride, GPUMatrixDynamic<bool> a byte array).
struct EditOperator {
	NsbEditOp pod{};
	virtual ~EditOperator() = default;
	// nerf_coords: NerfCoordinate per sample (7 floats); empty_mask is only ever set, like interpolate_tet / translate_in_box
	virtual void map_rays(void* stream, float* nerf_coords_dev, uint8_t* empty_mask_dev, uint32_t n_elements) const {
		check(nsb_map_rays_op(ctx(), m_index, nerf_coords_dev, empty_mask_dev, n_elements, stream), "nsb_map_rays_op");
	}
	virtual void map_positions(void* stream, float* nerf_pos_dev, uint32_t stride_floats, uint8_t* empty_mask_dev, uint32_t n_elements) const {
		check(nsb_map_positions(ctx(), m_index, nerf_pos_dev, stride_floats, empty_mask_dev, n_elements, stream), "nsb_map_positions");
	}
	virtual void compute_poisson_full_residuals(void* stream, uint32_t n_elements, const float* network_input_dev, float* sh_boundary_dev, float* out_density_boundary_dev,
	                                            float* residual_density_boundary_dev) const {
		check(nsb_poisson_residuals_op(ctx(), m_index, network_input_dev, n_elements, sh_boundary_dev, out_density_boundary_dev, residual_density_boundary_dev, stream), "nsb_poisson_residuals_op");
	}
	virtual void compute_poisson_residual_density(void* stream, uint32_t n_elements, const float* input_position_dev, uint32_t stride_floats, uint16_t* density_network_output_dev) const {
		check(nsb_poisson_residual_density(ctx(), m_index, input_position_dev, stride_floats, density_network_output_dev, n_elements, stream), "nsb_poisson_residual_density");
	}

private:
	friend class NerfTracer;
	NsbContext* ctx() const {
		if (!m_ctx || m_index < 0) throw std::runtime_error("EditOperator: not attached to a NerfTracer (add_edit_operator first)");
		return m_ctx;
	}
	NsbContext* m_ctx = nullptr;
	int32_t m_index = -1;
};
struct CageDeformation : EditOperator {
	CageDeformation() { pod.type = NSB_OP_CAGE; pod.residual_amplitude = 1.0f; }
};
struct AffineDuplication : EditOperator {
	AffineDuplication() { pod.type = NSB_OP_AFFINE; pod.scale[0] = pod.scale[1] = pod.scale[2] = 1.0f; pod.rotation[0] = pod.rotation[4] = pod.rotation[8] = 1.0f; }
};

class NerfTracer {
public:
	explicit NerfTracer(std::shared_ptr<Context> ctx) : m_ctx(std::move(ctx)) {}
	void add_edit_operator(std::shared_ptr<EditOperator> op) { m_edit_operators.push_back(std::move(op)); upload(); }
	void delete_edit_operator(size_t i) { m_edit_operators.erase(m_edit_operators.begin() + (long)i); upload(); }
	void reset_edit_operator() { m_edit_operators.clear(); upload(); }
	void update_edit_operators() { upload(); }  // after a gizmo drag changed an operator's arrays
	const std::vector<std::shared_ptr<EditOperator>>& edit_operators() const { return m_edit_operators; }
	bool m_poisson_target = false;

	// init_rays_from_camera + trace + shade in one call. Like NerfTracer::trace (:2998-3000) it synchronises the stream and returns n_hit;
	// synchronise = false keeps the frame asynchronous (returns 0; n_hit is in stats() later).
	uint32_t trace(const NsbFrame& frame, float* frame_buffer_dev, float* depth_buffer_dev, void* stream, bool synchronise = true) {
		NsbFrame f = frame;
		f.poisson_target = m_poisson_target ? 1 : 0;
		check(nsb_render(m_ctx->get(), &f, frame_buffer_dev, depth_buffer_dev, stream), "nsb_render");
		m_rendered = true;
		return synchronise ? (uint32_t)stats().n_hit : 0u;
	}
	// ---- per-edit work kept on the device (SURVEY.md §8f) ----
	// GrowingSelection::update_tet_mesh for operator i after a gizmo drag (growing_selection.cu:1615): no re-upload.
	void attach_mvc(size_t i, const float* mvc_weights, uint32_t n_cage_vertices) { check(nsb_cage_attach_mvc(m_ctx->get(), (int32_t)i, mvc_weights, n_cage_vertices), "nsb_cage_attach_mvc"); }
	void deform_cage(size_t i, const float* cage_vertices, uint32_t n_cage_vertices, void* stream) { check(nsb_cage_deform(m_ctx->get(), (int32_t)i, cage_vertices, n_cage_vertices, stream), "nsb_cage_deform"); }
	// TetMesh::vanish (tet_mesh.cu:251-363), the cage tool's "Vanish!" button: clears the cells operator i's tets cover in the context's
	// density grid and occupancy, stream-ordered. A later update_density_grid refills them from the network.
	void vanish_cage(size_t i, void* stream) { check(nsb_cage_vanish(m_ctx->get(), (int32_t)i, nullptr, stream), "nsb_cage_vanish"); }
	// GrowingSelection::interpolate_poisson_boundary (growing_selection.cu:2350-2398)
	void set_membrane(size_t i, const float* gamma, uint32_t n_cage_vertices, const float* d_in, const float* d_out, const float* shs_in, const float* shs_out, float amplitude, bool apply) {
		check(nsb_cage_set_membrane(m_ctx->get(), (int32_t)i, gamma, n_cage_vertices, d_in, d_out, shs_in, shs_out, amplitude, apply ? 1 : 0, nullptr, nullptr, nullptr), "nsb_cage_set_membrane");
	}
	// Testbed::update_density_grid_nerf_render (testbed_nerf.cu:3514-3520): the caller owns m_rng / density_grid_ema_step like Testbed does.
	void update_density_grid(const NsbGridUpdate& u, void* stream) { check(nsb_update_density_grid(m_ctx->get(), &u, stream), "nsb_update_density_grid"); }
	NsbRenderStats stats() const { NsbRenderStats s{}; check(nsb_get_stats(m_ctx->get(), &s), "nsb_get_stats"); return s; }
	void clear() {}  // the reference frees 4.6 GB of arena scratch here (:3074-3076); nothing to free

private:
	void upload() {
		std::vector<NsbEditOp> pods;
		for (size_t i = 0; i < m_edit_operators.size(); ++i) {
			m_edit_operators[i]->m_ctx = m_ctx->get();
			m_edit_operators[i]->m_index = (int32_t)i;
			pods.push_back(m_edit_operators[i]->pod);
		}
		check(nsb_set_edit_ops(m_ctx->get(), pods.empty() ? nullptr : pods.data(), (int32_t)pods.size()), "nsb_set_edit_ops");
	}
	std::shared_ptr<Context> m_ctx;
	std::vector<std::shared_ptr<EditOperator>> m_edit_operators;
	bool m_rendered = false;
};

// Testbed::render_nerf: the caller fills NsbFrame from the Testbed members listed at testbed_nerf.cu:3082-3138.
inline uint32_t render_nerf(NerfTracer& tracer, const NsbFrame& frame, float* frame_buffer_dev, float* depth_buffer_dev, bool apply_operators, void* stream, bool synchronise = false) {
	NsbFrame f = frame;
	f.apply_operators = apply_operators ? 1 : 0;
	return tracer.trace(f, frame_buffer_dev, depth_buffer_dev, stream, synchronise);
}

// CameraKeyframe (camera_path.h:30-62), Eigen-free: R is the quaternion (x, y, z, w). The arithmetic is float, in the order of Eigen's
// Quaternionf / Vector4f with SSE (a 4-vector's dot product sums (x0 + x2) + (x1 + x3)); compile without FMA contraction to keep it.
struct CameraKeyframe {
	float R[4] = {0.f, 0.f, 0.f, 1.f};
	float T[3] = {0.f, 0.f, 0.f};
	float slice = 0.f, scale = 1.f, fov = 50.625f, dof = 0.f;

	static float dot4(const float* a, const float* b) { return (a[0] * b[0] + a[2] * b[2]) + (a[1] * b[1] + a[3] * b[3]); }
	// Quaternionf(R).normalized().toRotationMatrix() and T, as a 3x4 column-major camera (NsbFrame::camera0)
	void m(float out[12]) const {
		const float n2 = dot4(R, R);
		float q[4] = {R[0], R[1], R[2], R[3]};
		if (n2 > 0.f) for (float& v : q) v = v / std::sqrt(n2);
		const float x = q[0], y = q[1], z = q[2], w = q[3];
		const float tx = 2.f * x, ty = 2.f * y, tz = 2.f * z;
		const float twx = tx * w, twy = ty * w, twz = tz * w, txx = tx * x, txy = ty * x, txz = tz * x, tyy = ty * y, tyz = tz * y, tzz = tz * z;
		const float r[9] = {1.f - (tyy + tzz), txy + twz, txz - twy,   // column 0
		                    txy - twz, 1.f - (txx + tzz), tyz + twx,   // column 1
		                    txz + twy, tyz - twx, 1.f - (txx + tyy)};  // column 2
		for (int i = 0; i < 9; ++i) out[i] = r[i];
		for (int i = 0; i < 3; ++i) out[9 + i] = T[i];
	}
	// CameraKeyframe(Matrix<float, 3, 4>, ...): Quaternionf(Matrix3f) (the trace and largest-diagonal branches); m column-major
	static CameraKeyframe from_matrix(const float m[12], float sl, float sc, float fv, float df) {
		CameraKeyframe k;
		auto at = [&](int r, int c) { return m[c * 3 + r]; };
		float t = (at(0, 0) + at(1, 1)) + at(2, 2);
		if (t > 0.f) {
			t = std::sqrt(t + 1.f);
			k.R[3] = 0.5f * t;
			t = 0.5f / t;
			k.R[0] = (at(2, 1) - at(1, 2)) * t;
			k.R[1] = (at(0, 2) - at(2, 0)) * t;
			k.R[2] = (at(1, 0) - at(0, 1)) * t;
		} else {
			int i = 0;
			if (at(1, 1) > at(0, 0)) i = 1;
			if (at(2, 2) > at(i, i)) i = 2;
			const int j = (i + 1) % 3, l = (j + 1) % 3;
			t = std::sqrt(at(i, i) - at(j, j) - at(l, l) + 1.f);
			k.R[i] = 0.5f * t;
			t = 0.5f / t;
			k.R[3] = (at(l, j) - at(j, l)) * t;
			k.R[j] = (at(j, i) + at(i, j)) * t;
			k.R[l] = (at(l, i) + at(i, l)) * t;
		}
		for (int a = 0; a < 3; ++a) k.T[a] = m[9 + a];
		k.slice = sl; k.scale = sc; k.fov = fv; k.dof = df;
		return k;
	}
	CameraKeyframe operator*(float f) const {
		CameraKeyframe k;
		for (int i = 0; i < 4; ++i) k.R[i] = R[i] * f;
		for (int i = 0; i < 3; ++i) k.T[i] = T[i] * f;
		k.slice = slice * f; k.scale = scale * f; k.fov = fov * f; k.dof = dof * f;
		return k;
	}
	CameraKeyframe operator+(const CameraKeyframe& rhs) const {  // the short path: flip rhs's quaternion when the dot product is negative
		const float s = dot4(rhs.R, R) < 0.f ? -1.f : 1.f;
		CameraKeyframe k;
		for (int i = 0; i < 4; ++i) k.R[i] = R[i] + s * rhs.R[i];
		for (int i = 0; i < 3; ++i) k.T[i] = T[i] + rhs.T[i];
		k.slice = slice + rhs.slice; k.scale = scale + rhs.scale; k.fov = fov + rhs.fov; k.dof = dof + rhs.dof;
		return k;
	}
};

// spline (camera_path.cu:52-70): the cubic B-spline branch the reference compiles (its Catmull-Rom branch is `if (0)`)
inline CameraKeyframe spline(float t, const CameraKeyframe& p0, const CameraKeyframe& p1, const CameraKeyframe& p2, const CameraKeyframe& p3) {
	const float tt = t * t, ttt = t * t * t;
	const float a = (1 - t) * (1 - t) * (1 - t) * (1.f / 6.f);
	const float b = (3.f * ttt - 6.f * tt + 4.f) * (1.f / 6.f);
	const float c = (-3.f * ttt + 3.f * tt + 3.f * t + 1.f) * (1.f / 6.f);
	const float d = ttt * (1.f / 6.f);
	return p0 * a + p1 * b + p2 * c + p3 * d;
}

struct CameraPath {
	std::vector<CameraKeyframe> m_keyframes;
	float m_playtime = 0.f;
	const CameraKeyframe& get_keyframe(int i) const { return m_keyframes[(size_t)std::min(std::max(i, 0), (int)m_keyframes.size() - 1)]; }
	CameraKeyframe eval_camera_path(float t) const {
		if (m_keyframes.empty()) return {};
		t *= (float)(m_keyframes.size() - 1);
		const int t1 = (int)std::floor(t);
		return spline(t - std::floor(t), get_keyframe(t1 - 1), get_keyframe(t1), get_keyframe(t1 + 1), get_keyframe(t1 + 2));
	}
};

// Testbed::marching_cubes (testbed_nerf.cu:4614-4649): density on the grid, marching cubes, normals and colours. The mesh stays in the
// context; the return value is the triangle count, like the reference's. density_dev: caller scratch of res[0]*res[1]*res[2] floats
// (res rounded up to multiples of 16 here, as the reference does); NULL meshes an existing grid given as grid_dev instead
// (GrowingSelection::extract_fine_mesh's selection grid, growing_selection.cu:2096-2162), then without shading.
struct Mesh { uint64_t n_vertices = 0, n_indices = 0; };
inline Mesh marching_cubes(Context& ctx, NsbGridQuery q, float* density_dev, float thresh, int32_t rgb_activation, bool linear_colors, void* stream,
                           const float* grid_dev = nullptr) {
	for (int a = 0; a < 3; ++a) q.res[a] = (q.res[a] + 15) / 16 * 16;
	Mesh m;
	if (!grid_dev) check(nsb_density_on_grid(ctx.get(), &q, density_dev, stream), "nsb_density_on_grid");
	check(nsb_marching_cubes(ctx.get(), grid_dev ? grid_dev : density_dev, q.res, q.aabb_min, q.aabb_max, thresh, &m.n_vertices, &m.n_indices, stream),
	      "nsb_marching_cubes");
	if (!grid_dev) check(nsb_mesh_shade(ctx.get(), q.train_aabb_min, q.train_aabb_max, rgb_activation, linear_colors ? 1 : 0, stream), "nsb_mesh_shade");
	return m;
}

// Testbed::optimise_mesh_step (testbed_nerf.cu:4470-4513) on the context's mesh, with m_mesh's thresh and amounts in `p`.
inline void optimise_mesh_step(Context& ctx, const NsbMeshOptimise& p, uint32_t n_steps, void* stream) {
	check(nsb_mesh_optimise(ctx.get(), &p, n_steps, stream), "nsb_mesh_optimise");
}

// Testbed::get_rgba_on_grid (testbed_nerf.cu:4588-4612): premultiplied RGBA of the field seen from ray_dir at the grid points of q (the
// reference samples m_render_aabb; q.res as the reference passes it, multiples of 16) into caller device memory (float4 per point).
inline void get_rgba_on_grid(Context& ctx, const NsbGridQuery& q, const float ray_dir[3], int32_t rgb_activation, int32_t density_activation, float* rgba_dev,
                             void* stream) {
	check(nsb_rgba_on_grid(ctx.get(), &q, ray_dir, rgb_activation, density_activation, rgba_dev, stream), "nsb_rgba_on_grid");
}

// scripts/run.py's --test_transforms block (run.py:215-302) on device frames: read_image's ground truth from decoded 8-bit pixels (with
// run.py's sRGB blend when srgb_blend), then compute_error("MSE") and compute_error("SSIM") of a rendered frame against it. mse_ssim_dev
// (2 floats) stays on the device; the maps are optional (nullptr).
inline void reference_image(Context& ctx, const uint8_t* pixels_dev, int32_t w, int32_t h, int32_t n_channels, bool srgb_blend, const float background[4],
                            float* rgba_dev, void* stream) {
	check(nsb_reference_image(ctx.get(), pixels_dev, w, h, n_channels, srgb_blend ? 1 : 0, background, rgba_dev, stream), "nsb_reference_image");
}
inline void image_metrics(Context& ctx, const float* image_dev, const float* ref_dev, int32_t w, int32_t h, float* mse_ssim_dev, void* stream,
                          float* mse_map_dev = nullptr, float* ssim_map_dev = nullptr) {
	check(nsb_image_metrics(ctx.get(), image_dev, ref_dev, w, h, mse_ssim_dev, mse_map_dev, ssim_map_dev, stream), "nsb_image_metrics");
}

#ifdef NSB_HOST_HAVE_CUDART
namespace detail {
struct CudaFree { void operator()(void* p) const { cudaFree(p); } };
inline std::unique_ptr<void, CudaFree> device_alloc(size_t bytes) {
	void* p = nullptr;
	if (cudaMalloc(&p, bytes) != cudaSuccess) throw std::runtime_error("cudaMalloc failed");
	return std::unique_ptr<void, CudaFree>(p);
}
inline void download(void* dst, const void* src, size_t bytes, void* stream) {
	if (cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream) != cudaSuccess || cudaStreamSynchronize((cudaStream_t)stream) != cudaSuccess)
		throw std::runtime_error("device-to-host copy failed");
}
}  // namespace detail

// save_density_grid_to_png (marching_cubes.cu:898-974) up to its stbi_write_png(filename, w, h, 1, pixels.data(), w) and its log line,
// for a device float grid such as Testbed::get_density_on_grid's (compute_and_save_png_slices, testbed.cu:345-366).
struct DensityPng {
	uint32_t w = 0, h = 0;
	std::vector<uint8_t> pixels;  // w * h
	uint64_t n_zero_x_voxels = 0, n_lattice_near_zero_x = 0;
};
inline DensityPng density_png(Context& ctx, const float* density_dev, const int32_t res[3], float thresh, float density_range, bool swap_y_z, void* stream) {
	DensityPng p;
	check(nsb_density_png_extent(res, swap_y_z ? 1 : 0, &p.w, &p.h), "nsb_density_png_extent");
	p.pixels.resize((size_t)p.w * p.h);
	const size_t counts_at = (p.pixels.size() + 7) & ~size_t(7);  // the counts after the pixels, 8-byte aligned
	auto px = detail::device_alloc(counts_at + 2 * sizeof(uint64_t));
	uint64_t* counts = reinterpret_cast<uint64_t*>(static_cast<uint8_t*>(px.get()) + counts_at);
	check(nsb_density_png(ctx.get(), density_dev, res, thresh, density_range, swap_y_z ? 1 : 0, static_cast<uint8_t*>(px.get()), counts, stream), "nsb_density_png");
	uint64_t c[2];
	detail::download(p.pixels.data(), px.get(), p.pixels.size(), stream);
	detail::download(c, counts, sizeof(c), stream);
	p.n_zero_x_voxels = c[0];
	p.n_lattice_near_zero_x = c[1];
	return p;
}

// save_rgba_grid_to_png_sequence (marching_cubes.cu:979-1015) up to its stbi_write_png(path/%04d_<w>x<h>.png, w, h, 4, slice z, w * 4),
// for a device float4 grid such as get_rgba_on_grid's.
struct RgbaPng {
	uint32_t w = 0, h = 0, n_slices = 0;
	std::vector<uint8_t> pixels;  // n_slices images of w * h * 4 bytes, back to back
	const uint8_t* slice(uint32_t z) const { return pixels.data() + (size_t)z * w * h * 4; }
};
inline RgbaPng rgba_png(Context& ctx, const float* rgba_dev, const int32_t res[3], bool swap_y_z, void* stream) {
	RgbaPng p;
	p.w = (uint32_t)res[0];
	p.h = (uint32_t)(swap_y_z ? res[2] : res[1]);
	p.n_slices = (uint32_t)(swap_y_z ? res[1] : res[2]);
	p.pixels.resize((size_t)p.w * p.h * p.n_slices * 4);
	auto px = detail::device_alloc(p.pixels.size());
	check(nsb_rgba_png(ctx.get(), rgba_dev, res, swap_y_z ? 1 : 0, static_cast<uint8_t*>(px.get()), stream), "nsb_rgba_png");
	detail::download(p.pixels.data(), px.get(), p.pixels.size(), stream);
	return p;
}
// Testbed::render_to_cpu (python_api.cu:129-175) once its sub-frames are known: every sub-frame rendered and accumulated, one tonemap, the
// float4 frame copied to rgba_host (width * height * 4 floats) and the stream synchronised. accumulate_dev / out_rgba_dev: caller device
// buffers of the frame's size (the reference's m_windowless_render_surface).
inline void render_to_cpu(Context& ctx, const std::vector<NsbFrame>& sub_frames, const NsbTonemap& tm, float* accumulate_dev, float* out_rgba_dev,
                          float* rgba_host, void* stream) {
	if (sub_frames.empty()) throw std::runtime_error("render_to_cpu: no sub-frames");
	check(nsb_render_accumulate(ctx.get(), sub_frames.data(), (uint32_t)sub_frames.size(), &tm, accumulate_dev, out_rgba_dev, stream), "nsb_render_accumulate");
	detail::download(rgba_host, out_rgba_dev, (size_t)sub_frames[0].width * sub_frames[0].height * 16, stream);
}
#endif  // NSB_HOST_HAVE_CUDART

}  // namespace ngp_b200
