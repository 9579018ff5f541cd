// ref_mesh_driver_cuda.cu — the reference's OWN mesh-extraction code (marching_cubes.cu, the grid / colour kernels of testbed_nerf.cu),
// compiled by nvcc for sm_90a into oracle/_ref/libnerfshop_ref_mesh_cuda.so by oracle/ref_mesh_build.py. TEST INFRASTRUCTURE ONLY.
// Host pointers in and out; each call copies its inputs to the device, runs the reference's kernel or host function as it is, and copies
// the result back. The network (tiny-cuda-nn, absent) is not here: the caller runs nsb_density / nsb_inference between the calls.
#include <tiny-cuda-nn/common.h>
#include <tiny-cuda-nn/gpu_matrix.h>
#include <tiny-cuda-nn/gpu_memory.h>
#include <tinylogger/tinylogger.h>

#include <cstdio>
#include <memory>
#include <stdexcept>
#include <vector>

#include <neural-graphics-primitives/common.h>
#include <neural-graphics-primitives/common_device.cuh>
#include <neural-graphics-primitives/common_nerf.h>
#include <neural-graphics-primitives/bounding_box.cuh>
#include <neural-graphics-primitives/nerf.h>

#include <common_nerf.cu>  // /root/reference/src/common_nerf.cu, whole file

#include <filesystem/path.h>  // oracle/ref_shim_mesh
#include <stb_image/stb_image_write.h>

namespace tcnn {
// tcnn::allocate_workspace(stream, bytes).data(): marching_cubes_gpu's vertex-index grid
struct MeshWorkspace {
	std::shared_ptr<void> p;
	void* data() const { return p.get(); }
};
inline MeshWorkspace allocate_workspace(cudaStream_t, size_t bytes) {
	void* q = nullptr;
	CUDA_CHECK_THROW(cudaMalloc(&q, bytes));
	return MeshWorkspace{std::shared_ptr<void>(q, [](void* x) { cudaFree(x); })};
}
}  // namespace tcnn

NGP_NAMESPACE_BEGIN
using namespace Eigen;
using namespace tcnn;
namespace fs = filesystem;
#include "marching_cubes_mesh.inc"
#include "testbed_nerf_mesh.inc"
NGP_NAMESPACE_END

using namespace ngp;
static_assert(sizeof(Eigen::Vector3f) == 12, "Vector3f rows are 3 floats");

namespace {
BoundingBox box(const float* a) { return BoundingBox{Eigen::Vector3f{a[0], a[1], a[2]}, Eigen::Vector3f{a[3], a[4], a[5]}}; }
template <typename T> tcnn::GPUMemory<T> up(const void* h, size_t n) {
	tcnn::GPUMemory<T> m(n);
	if (n) CUDA_CHECK_THROW(cudaMemcpy(m.data(), h, n * sizeof(T), cudaMemcpyHostToDevice));
	return m;
}
template <typename T> void down(void* h, const tcnn::GPUMemory<T>& m, size_t n) {
	CUDA_CHECK_THROW(cudaDeviceSynchronize());
	if (n) CUDA_CHECK_THROW(cudaMemcpy(h, m.data(), n * sizeof(T), cudaMemcpyDeviceToHost));
}
tcnn::GPUMemory<Eigen::Vector3f> g_verts;
tcnn::GPUMemory<uint32_t> g_indices;
template <typename F> int guarded(F f) {
	try {
		f();
		CUDA_CHECK_THROW(cudaDeviceSynchronize());
		return 0;
	} catch (const std::exception& e) {
		fprintf(stderr, "ref mesh: %s\n", e.what());
		return 1;
	}
}
}  // namespace

extern "C" {
uint32_t ref_mesh_position_floats() { return sizeof(NerfPosition) / sizeof(float); }
uint32_t ref_mesh_coordinate_floats() { return sizeof(NerfCoordinate) / sizeof(float); }

int ref_mesh_res(uint32_t res_1d, const float* aabb, int32_t* out) {
	return guarded([&] { Eigen::Vector3i r = get_marching_cubes_res(res_1d, box(aabb)); out[0] = r.x(); out[1] = r.y(); out[2] = r.z(); });
}
// generate_grid_samples_nerf_uniform with Testbed::get_density_on_grid's launch (testbed_nerf.cu:4560-4563): NerfPosition rows
int ref_mesh_grid_positions(const int32_t* res, const float* render_aabb, const float* train_aabb, float* pos_out) {
	return guarded([&] {
		const Eigen::Vector3i r{res[0], res[1], res[2]};
		const uint32_t n = (uint32_t)(res[0] * res[1] * res[2]);
		tcnn::GPUMemory<NerfPosition> pos(n);
		const dim3 threads = {16, 8, 1};
		const dim3 blocks = {div_round_up((uint32_t)r.x(), threads.x), div_round_up((uint32_t)r.y(), threads.y), div_round_up((uint32_t)r.z(), threads.z)};
		generate_grid_samples_nerf_uniform<<<blocks, threads>>>(r, 0u, box(render_aabb), box(train_aabb), pos.data());
		down(pos_out, pos, n);
	});
}
// grid_samples_half_to_float over n samples: mlp = density row of the network output (fp16), grid = 5 x 128^3 floats or NULL
int ref_mesh_half_to_float(uint32_t n, const float* train_aabb, const uint16_t* mlp, const float* pos, const float* grid, float* out) {
	return guarded([&] {
		auto d_mlp = up<tcnn::network_precision_t>(mlp, n);
		auto d_pos = up<NerfPosition>(pos, n);
		tcnn::GPUMemory<float> d_grid;
		if (grid) d_grid = up<float>(grid, (size_t)NERF_GRIDVOLUME() * NERF_CASCADES());
		tcnn::GPUMemory<float> d_out(n);
		linear_kernel(grid_samples_half_to_float, 0, nullptr, n, box(train_aabb), d_out.data(), d_mlp.data(), ENerfActivation::Exponential, d_pos.data(),
		              grid ? (const float*)d_grid.data() : nullptr);
		down(out, d_out, n);
	});
}
// marching_cubes_gpu; the result stays here for ref_mesh_get (rows = vertices rounded up to 128)
// ms (may be NULL): device time of marching_cubes_gpu alone (CUDA events; the density upload is outside)
int ref_mesh_marching_cubes(const float* aabb, const int32_t* res, float thresh, const float* density, uint64_t* n_rows, uint64_t* n_indices, float* ms) {
	return guarded([&] {
		auto d = up<float>(density, (size_t)res[0] * res[1] * res[2]);
		cudaEvent_t e0, e1;
		CUDA_CHECK_THROW(cudaEventCreate(&e0));
		CUDA_CHECK_THROW(cudaEventCreate(&e1));
		CUDA_CHECK_THROW(cudaEventRecord(e0));
		marching_cubes_gpu(nullptr, box(aabb), Eigen::Vector3i{res[0], res[1], res[2]}, thresh, d, g_verts, g_indices);
		CUDA_CHECK_THROW(cudaEventRecord(e1));
		CUDA_CHECK_THROW(cudaEventSynchronize(e1));
		if (ms) CUDA_CHECK_THROW(cudaEventElapsedTime(ms, e0, e1));
		cudaEventDestroy(e0);
		cudaEventDestroy(e1);
		*n_rows = g_verts.size();
		*n_indices = g_indices.size();
	});
}
int ref_mesh_get(float* verts, uint32_t* indices) {
	return guarded([&] { down(verts, g_verts, g_verts.size()); down(indices, g_indices, g_indices.size()); });
}
// compute_mesh_1ring's normals (float atomics: order-dependent in the last bits)
int ref_mesh_normals(uint32_t n_verts, const float* verts, uint32_t n_indices, const uint32_t* indices, float* normals) {
	return guarded([&] {
		auto v = up<Eigen::Vector3f>(verts, n_verts);
		auto i = up<uint32_t>(indices, n_indices);
		tcnn::GPUMemory<Eigen::Vector4f> smoothed;
		tcnn::GPUMemory<Eigen::Vector3f> nrm;
		compute_mesh_1ring(v, i, smoothed, nrm);
		down(normals, nrm, n_verts);
	});
}
// generate_nerf_network_inputs_from_positions (no extra dims): NerfCoordinate rows
int ref_mesh_color_inputs(uint32_t n, const float* train_aabb, const float* pos, float* coords) {
	return guarded([&] {
		auto p = up<Eigen::Vector3f>(pos, n);
		tcnn::GPUMemory<NerfCoordinate> c(n);
		linear_kernel(generate_nerf_network_inputs_from_positions, 0, nullptr, n, box(train_aabb), p.data(), PitchedPtr<NerfCoordinate>(c.data(), 1, 0, 0),
		              Eigen::Vector3f{0.f, 0.f, 1.f});
		down(coords, c, n);
	});
}
// extract_srgb_with_activation: rgbd = n x 4 floats (the network output as m_network->inference writes it)
int ref_mesh_srgb(uint32_t n, const float* rgbd, int32_t rgb_activation, int32_t linear_colors, float* rgb) {
	return guarded([&] {
		auto in = up<float>(rgbd, (size_t)n * 4);
		tcnn::GPUMemory<float> out((size_t)n * 3);
		linear_kernel(extract_srgb_with_activation, 0, nullptr, n * 3, 3u, in.data(), out.data(), (ENerfActivation)rgb_activation, linear_colors != 0);
		down(rgb, out, (size_t)n * 3);
	});
}
int ref_mesh_save(const char* path, uint32_t n_rows, const float* verts, const float* normals, const float* colors, uint32_t n_indices, const uint32_t* indices,
                  float nerf_scale, const float* nerf_offset) {
	return guarded([&] {
		auto v = up<Eigen::Vector3f>(verts, n_rows);
		auto nn = up<Eigen::Vector3f>(normals, n_rows);
		auto c = up<Eigen::Vector3f>(colors, n_rows);
		auto i = up<uint32_t>(indices, n_indices);
		save_mesh(v, nn, c, i, path, false, nerf_scale, Eigen::Vector3f{nerf_offset[0], nerf_offset[1], nerf_offset[2]});
	});
}
}
