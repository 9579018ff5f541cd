// ref_mesh_opt_driver_cuda.cu — the reference's OWN mesh optimisation gradient (compute_mesh_1ring, compute_mesh_opt_gradients of
// marching_cubes.cu), compiled by nvcc for sm_90a into oracle/_ref/libnerfshop_ref_mesh_opt_cuda.so by oracle/ref_mesh_opt_build.py.
// TEST INFRASTRUCTURE ONLY. Host pointers in and out, as ref_mesh_driver_cuda.cu. The network (tiny-cuda-nn, absent) and the optimiser
// (tcnn Adam, absent) are not here: the caller runs nsb_density_gradient before and the restated Adam after.
#include <tiny-cuda-nn/common.h>
#include <tiny-cuda-nn/gpu_memory.h>
#include <tinylogger/tinylogger.h>

#include <cstdio>
#include <stdexcept>

#include <neural-graphics-primitives/common.h>
#include <neural-graphics-primitives/common_device.cuh>

NGP_NAMESPACE_BEGIN
using namespace Eigen;
using namespace tcnn;
#include "marching_cubes_opt.inc"
NGP_NAMESPACE_END

using namespace ngp;
static_assert(sizeof(Eigen::Vector3f) == 12, "Vector3f rows are 3 floats");
static_assert(sizeof(Eigen::Vector4f) == 16, "Vector4f rows are 4 floats");

namespace {
template <typename T> tcnn::GPUMemory<T> up(const void* h, size_t n) {
	tcnn::GPUMemory<T> m(n);
	if (n) CUDA_CHECK_THROW(cudaMemcpy(m.data(), h, n * sizeof(T), cudaMemcpyHostToDevice));
	return m;
}
template <typename T> void down(void* h, const tcnn::GPUMemory<T>& m, size_t n) {
	CUDA_CHECK_THROW(cudaDeviceSynchronize());
	if (n) CUDA_CHECK_THROW(cudaMemcpy(h, m.data(), n * sizeof(T), cudaMemcpyDeviceToHost));
}
template <typename F> int guarded(F f) {
	try {
		f();
		CUDA_CHECK_THROW(cudaDeviceSynchronize());
		return 0;
	} catch (const std::exception& e) {
		fprintf(stderr, "ref mesh opt: %s\n", e.what());
		return 1;
	}
}
}  // namespace

extern "C" {
// Testbed::optimise_mesh_step between the network and the optimiser (testbed_nerf.cu:4494-4508): compute_mesh_1ring of the vertex rows, then
// compute_mesh_opt_gradients with densities = the fp16 density row [n_verts] and input_gradients = rows of `grad_width` floats.
// Out: the opt gradient [n_verts x 3], the 1-ring sums [n_verts x 4] and normals [n_verts x 3] (float atomics: order-dependent in the last bits).
int ref_mesh_opt_gradients(uint32_t n_verts, const float* verts, uint32_t n_indices, const uint32_t* indices, const uint16_t* densities,
                           uint32_t grad_width, const float* input_gradients, float thresh, float k_smooth, float k_density, float k_inflate,
                           float* grad_out, float* smoothed_out, float* normals_out) {
	return guarded([&] {
		auto v = up<Eigen::Vector3f>(verts, n_verts);
		auto i = up<uint32_t>(indices, n_indices);
		auto d = up<tcnn::network_precision_t>(densities, n_verts);
		auto g = up<float>(input_gradients, (size_t)n_verts * grad_width);
		tcnn::GPUMemory<Eigen::Vector4f> smoothed;
		tcnn::GPUMemory<Eigen::Vector3f> nrm;
		compute_mesh_1ring(v, i, smoothed, nrm);
		tcnn::GPUMemory<Eigen::Vector3f> out(n_verts);
		compute_mesh_opt_gradients(thresh, v, nrm, smoothed, d.data(), grad_width, g.data(), out, k_smooth, k_density, k_inflate);
		down(grad_out, out, n_verts);
		down(smoothed_out, smoothed, n_verts);
		down(normals_out, nrm, n_verts);
	});
}
}  // extern "C"
