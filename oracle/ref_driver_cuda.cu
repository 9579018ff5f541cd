// ref_driver_cuda.cu — the reference's OWN CUDA render path, compiled by nvcc for sm_90a (oracle/_ref/libnerfshop_ref_cuda.so).
//
// TEST / BASELINE INFRASTRUCTURE ONLY. Same reference sources as oracle/ref_driver.cpp (see ref_build.py EXTRACTS and
// ref_common.inl) — Testbed::render_nerf, NerfTracer::{init_rays_from_camera, trace, enlarge}, every kernel they launch, the
// cage / affine operator kernels — but here they are real __global__ kernels launched on the GPU by the reference's own host
// loop (compaction with global atomics, a host sync per round, two inferences per round, 1-8 samples per ray per round).
// The one thing that is not the reference's: tiny-cuda-nn's network (absent submodule). NerfNetwork::inference_mixed_precision
// forwards to a C function pointer with nsb_inference's signature, so the caller can plug in this repository's encode + MLP
// kernel; the reference arm therefore runs OUR fast network inside THEIR pipeline ("ref_cuda" in bench.py's gpu_baseline).
// Used for (1) bit-exact parity of ray generation / occupancy stepping / deformation against what nvcc makes of the reference's
// expressions (FMA contraction included), (2) the GPU baseline the north star asks to be timed next to the native path.
#include <tiny-cuda-nn/common.h>
#include <tiny-cuda-nn/gpu_matrix.h>
#include <tiny-cuda-nn/gpu_memory.h>
#include <tiny-cuda-nn/random.h>

#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <queue>
#include <tuple>

#include <neural-graphics-primitives/common.h>
#include <neural-graphics-primitives/common_gl.h>  // oracle/ref_shim shadow
#include <neural-graphics-primitives/common_device.cuh>
#include <neural-graphics-primitives/common_nerf.h>
#include <neural-graphics-primitives/envmap.cuh>
#include <neural-graphics-primitives/random_val.cuh>
#include <neural-graphics-primitives/editing/edit_operator.h>
#include <neural-graphics-primitives/editing/tools/affine_bounding_box.cuh>
#include <neural-graphics-primitives/editing/tools/selection_utils.h>

#include <common_nerf.cu>  // /root/reference/src/common_nerf.cu, whole file

#include "../include/nerfshop_b200.h"

// tcnn's GPUMemoryArena keeps freed workspace for the next frame; so does this (size-keyed free lists), otherwise the reference
// arm would pay a cudaMalloc/cudaFree of its 4.6 GB scratch every frame, which the real reference does not.
namespace {
std::mutex g_pool_mutex;
std::multimap<size_t, void*> g_pool;
std::shared_ptr<void> nsb_ref_alloc(size_t bytes) {
	void* p = nullptr;
	{
		std::lock_guard<std::mutex> lock(g_pool_mutex);
		auto it = g_pool.find(bytes);
		if (it != g_pool.end()) { p = it->second; g_pool.erase(it); }
	}
	if (!p) CUDA_CHECK_THROW(cudaMalloc(&p, bytes));
	return std::shared_ptr<void>(p, [bytes](void* q) { std::lock_guard<std::mutex> lock(g_pool_mutex); g_pool.emplace(bytes, q); });
}
void pool_release() {
	std::lock_guard<std::mutex> lock(g_pool_mutex);
	for (auto& kv : g_pool) cudaFree(kv.second);
	g_pool.clear();
}
}  // namespace
#include "ref_common.inl"

using namespace ngp;

static Eigen::Matrix<float, 3, 4> cam34(const float* m) { Eigen::Matrix<float, 3, 4> r; memcpy(r.data(), m, 12 * sizeof(float)); return r; }

struct RefCuScene {
	std::vector<void*> owned;
	std::vector<NsbEditOp> ops;  // pointers are DEVICE pointers
	Testbed tb;
	template <typename T> const T* up(const T* host, size_t n) {
		if (!host || !n) return nullptr;
		void* d = nullptr;
		CUDA_CHECK_THROW(cudaMalloc(&d, n * sizeof(T)));
		CUDA_CHECK_THROW(cudaMemcpy(d, host, n * sizeof(T), cudaMemcpyHostToDevice));
		owned.push_back(d);
		return (const T*)d;
	}
	~RefCuScene() { for (void* p : owned) cudaFree(p); }
};

static void configure(RefCuScene& sc, const NsbFrame* f) {
	Testbed& tb = sc.tb;
	tb.m_render_mode = (ERenderMode)f->render_mode;
	tb.m_snap_to_pixel_centers = f->snap_to_pixel_centers != 0;
	tb.m_render_aabb = bb(f->render_aabb_min, f->render_aabb_max);
	tb.m_aabb = bb(f->train_aabb_min, f->train_aabb_max);
	tb.m_nerf.show_accel = f->show_accel ? f->min_mip : -1;  // the reference derives min_mip from show_accel; without the override min_mip is 0
	tb.m_nerf.cone_angle_constant = f->cone_angle_constant;
	tb.m_nerf.training.dataset.scale = 1.0f / f->depth_scale;
	tb.m_nerf.training.linear_colors = f->linear_colors != 0;
	tb.m_nerf.rgb_activation = (ENerfActivation)f->rgb_activation;
	tb.m_nerf.density_activation = (ENerfActivation)f->density_activation;
	tb.m_nerf.rendering_min_transmittance = f->min_transmittance;
	tb.m_nerf.tracer.m_poisson_target = f->poisson_target != 0;
	set_frame_extras(tb, f);  // ABI 3: general camera, glow, environment / distortion maps (device pointers)
}

extern "C" {

void* refcu_create(const uint8_t* bitfield_host, const NsbEditOp* ops, int n_ops) {
	try {
		auto sc = std::make_unique<RefCuScene>();
		sc->tb.m_nerf.density_grid_bitfield.copy_from_host(bitfield_host, NSB_BITFIELD_BYTES);
		for (int i = 0; i < n_ops; ++i) {
			NsbEditOp o = ops[i];
			if (o.type == NSB_OP_CAGE) {
				o.tet_lut_offsets = sc->up(ops[i].tet_lut_offsets, (size_t)NSB_GRID_CELLS + 1);
				o.tet_lut_idx = sc->up(ops[i].tet_lut_idx, o.n_lut_idx);
				o.tets = sc->up(ops[i].tets, 4 * (size_t)o.n_tets);
				o.vertices = sc->up(ops[i].vertices, 3 * (size_t)o.n_vertices);
				o.original_vertices = sc->up(ops[i].original_vertices, 3 * (size_t)o.n_vertices);
				o.local_rotations = sc->up(ops[i].local_rotations, 9 * (size_t)o.n_tets);
				o.original_bitfield = sc->up(ops[i].original_bitfield, NSB_BITFIELD_BYTES);
				o.boundary_shs = sc->up(ops[i].boundary_shs, 27 * (size_t)o.n_vertices);
				o.boundary_outside_density = sc->up(ops[i].boundary_outside_density, o.n_vertices);
				o.boundary_residual_density = sc->up(ops[i].boundary_residual_density, o.n_vertices);
			}
			sc->ops.push_back(o);
			sc->tb.m_nerf.tracer.add_edit_operator(make_op(o));
		}
		return sc.release();
	} catch (const std::exception& e) {
		fprintf(stderr, "refcu_create: %s\n", e.what());
		return nullptr;
	}
}
void refcu_destroy(void* scene) { delete (RefCuScene*)scene; pool_release(); }

// Testbed::render_nerf of the reference on the GPU. fb_dev / depth_dev: caller-owned device buffers (float4[W*H], float[W*H]).
int refcu_render(void* scene, const NsbFrame* f, void* inference_fn, void* inference_ctx, float* fb_dev, float* depth_dev, void* stream, uint64_t* stats /*3: n_inferred, n_calls, rays*/) {
	try {
		RefCuScene& sc = *(RefCuScene*)scene;
		configure(sc, f);
		NerfNetwork<network_precision_t> net;
		net.fn = (ref_inference_fn)inference_fn;
		net.user = inference_ctx;
		CudaRenderBuffer rb;
		rb.res = Vector2i(f->width, f->height); rb.m_spp = f->spp_index; rb.fb = (Array4f*)fb_dev; rb.depth = depth_dev;
		sc.tb.render_nerf(net, rb, rb.res, Vector2f(f->focal_length[0], f->focal_length[1]), cam34(f->camera0), cam34(f->camera1),
		                  Vector4f(f->rolling_shutter[0], f->rolling_shutter[1], f->rolling_shutter[2], f->rolling_shutter[3]), Vector2f(f->screen_center[0], f->screen_center[1]),
		                  f->apply_operators != 0, (cudaStream_t)stream);
		if (stats) { stats[0] = net.n_inferred; stats[1] = net.n_calls; stats[2] = (uint64_t)f->width * f->height; }
		return 0;
	} catch (const std::exception& e) {
		fprintf(stderr, "refcu_render: %s\n", e.what());
		return 1;
	}
}

// Ray generation + occupancy march with the reference's kernels on the GPU: init_rays_from_camera (init_rays_with_payload_kernel_nerf
// + advance_pos_nerf), then generate_next_nerf_network_inputs with n_steps = 1 over ALL rays, max_samples times, no compaction.
// Outputs for the listed pixels (host arrays): rec [n_pixels][max_samples][8] = NerfCoordinate (7) + payload.t after the step,
// ray [n_pixels][8] = origin, dir, t after advance_pos (first sample), alive flag after advance_pos; count [n_pixels].
int refcu_march_trace(void* scene, const NsbFrame* f, const uint32_t* pixels, uint32_t n_pixels, uint32_t max_samples, float* rec, float* ray, uint32_t* count) {
	try {
		RefCuScene& sc = *(RefCuScene*)scene;
		configure(sc, f);
		Testbed& tb = sc.tb;
		const uint32_t W = (uint32_t)f->width, H = (uint32_t)f->height, N = W * H;
		GPUMemory<Array4f> fb(N); GPUMemory<float> depth(N);
		fb.memset(0);
		tb.m_nerf.tracer.init_rays_from_camera(f->spp_index, 16, 0, Vector2i((int)W, (int)H), Vector2f(f->focal_length[0], f->focal_length[1]), cam34(f->camera0), cam34(f->camera1),
		                                        Vector4f(f->rolling_shutter[0], f->rolling_shutter[1], f->rolling_shutter[2], f->rolling_shutter[3]),
		                                        Vector2f(f->screen_center[0], f->screen_center[1]), tb.m_snap_to_pixel_centers, tb.m_render_aabb, tb.m_slice_plane_z + tb.m_scale, tb.m_dof, frame_camera_distortion(f), nullptr,
		                                        Vector2i::Zero(), f->distortion_dev, Vector2i(f->distortion_resolution[0], f->distortion_resolution[1]), fb.data(), depth.data(), tb.m_nerf.density_grid_bitfield.data(), tb.m_nerf.show_accel,
		                                        tb.m_nerf.cone_angle_constant, (ERenderMode)f->render_mode, nullptr);
		NerfPayload* payloads_dev = tb.m_nerf.tracer.rays_init().payload;
		std::vector<NerfPayload> payloads(N);
		CUDA_CHECK_THROW(cudaMemcpy(payloads.data(), payloads_dev, N * sizeof(NerfPayload), cudaMemcpyDeviceToHost));
		for (uint32_t k = 0; k < n_pixels; ++k) {
			const NerfPayload& p = payloads[pixels[k]];
			float* rr = ray + 8 * (size_t)k;
			rr[0] = p.origin.x(); rr[1] = p.origin.y(); rr[2] = p.origin.z(); rr[3] = p.dir.x(); rr[4] = p.dir.y(); rr[5] = p.dir.z(); rr[6] = p.t; rr[7] = p.alive ? 1.0f : 0.0f;
			count[k] = 0;
		}
		GPUMemory<NerfCoordinate> input_dev(N);
		std::vector<float> input((size_t)N * 7);
		std::vector<uint8_t> done(n_pixels, 0);
		for (uint32_t s = 0; s < max_samples; ++s) {
			linear_kernel(generate_next_nerf_network_inputs, 0, nullptr, N, tb.m_render_aabb, tb.m_aabb, Vector2f(f->focal_length[0], f->focal_length[1]), cam34(f->camera1).col(2), payloads_dev,
			              PitchedPtr<NerfCoordinate>(input_dev.data(), 1, 0, 0), 1u, (const uint8_t*)tb.m_nerf.density_grid_bitfield.data(), (uint32_t)(f->min_mip > 0 ? f->min_mip : 0),
			              tb.m_nerf.cone_angle_constant, Vector3f(Vector3f::Zero()));
			CUDA_CHECK_THROW(cudaMemcpy(payloads.data(), payloads_dev, N * sizeof(NerfPayload), cudaMemcpyDeviceToHost));
			CUDA_CHECK_THROW(cudaMemcpy(input.data(), input_dev.data(), (size_t)N * 7 * sizeof(float), cudaMemcpyDeviceToHost));
			for (uint32_t k = 0; k < n_pixels; ++k) {
				const NerfPayload& p = payloads[pixels[k]];
				if (done[k] || !p.alive) continue;
				if (p.n_steps == 0) { done[k] = 1; continue; }  // left the render aabb (the kernel keeps returning early from now on)
				float* o = rec + ((size_t)k * max_samples + count[k]) * 8;
				memcpy(o, input.data() + (size_t)pixels[k] * 7, 7 * sizeof(float));
				o[7] = p.t;
				++count[k];
			}
		}
		tb.m_nerf.tracer.clear();
		return 0;
	} catch (const std::exception& e) {
		fprintf(stderr, "refcu_march_trace: %s\n", e.what());
		return 1;
	}
}

// EditOperator::map_rays over a flat host batch, all operators of the scene in reverse list order (testbed_nerf.cu:2896-2904)
int refcu_map_rays(void* scene, float* coords /*7 per sample, host*/, uint8_t* empty_mask /*host*/, uint32_t n) {
	try {
		RefCuScene& sc = *(RefCuScene*)scene;
		GPUMemory<float> c((size_t)n * 7);
		c.copy_from_host(coords, (size_t)n * 7);
		GPUMatrix<bool> mask(1, n);
		CUDA_CHECK_THROW(cudaMemset(mask.data(), 0, n));
		auto& ops = sc.tb.m_nerf.tracer.edit_operators();
		for (int i = (int)ops.size() - 1; i >= 0; --i) ops[i]->map_rays(nullptr, PitchedPtr<NerfCoordinate>((NerfCoordinate*)c.data(), 1, 0, 0), mask, n);
		c.copy_to_host(coords, (size_t)n * 7);
		static_assert(sizeof(bool) == 1, "bool mask bytes");
		CUDA_CHECK_THROW(cudaMemcpy(empty_mask, mask.data(), n, cudaMemcpyDeviceToHost));
		return 0;
	} catch (const std::exception& e) {
		fprintf(stderr, "refcu_map_rays: %s\n", e.what());
		return 1;
	}
}
int refcu_poisson_residuals(void* scene, const float* coords, uint32_t n, float* sh /*27 per*/, float* out_density, float* residual_density) {
	try {
		RefCuScene& sc = *(RefCuScene*)scene;
		GPUMemory<float> c((size_t)n * 7);
		c.copy_from_host(coords, (size_t)n * 7);
		std::vector<NerfPayload> ph(n);
		for (auto& p : ph) { p.n_steps = 1; p.alive = true; }
		GPUMemory<NerfPayload> payloads(n);
		payloads.copy_from_host(ph.data(), n);
		GPUMemory<SH9RGB> shs(n); GPUMemory<float> od(n), rd(n);
		shs.memset(0); od.memset(0); rd.memset(0);
		auto& ops = sc.tb.m_nerf.tracer.edit_operators();
		for (int i = (int)ops.size() - 1; i >= 0; --i)
			ops[i]->compute_poisson_full_residuals(nullptr, n, payloads.data(), PitchedPtr<NerfCoordinate>((NerfCoordinate*)c.data(), 1, 0, 0), shs.data(), od.data(), rd.data());
		CUDA_CHECK_THROW(cudaMemcpy(sh, shs.data(), (size_t)n * 27 * sizeof(float), cudaMemcpyDeviceToHost));
		od.copy_to_host(out_density, n);
		rd.copy_to_host(residual_density, n);
		return 0;
	} catch (const std::exception& e) {
		fprintf(stderr, "refcu_poisson_residuals: %s\n", e.what());
		return 1;
	}
}

}  // extern "C"
