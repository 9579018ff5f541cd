// ref_slices_driver_cuda.cu — the reference's OWN slice-export code (the RGBA grid kernels of testbed_nerf.cu, the PNG writers of
// marching_cubes.cu), compiled by nvcc for sm_90a into oracle/_ref/libnerfshop_ref_slices_cuda.so by oracle/ref_slices_build.py.
// TEST INFRASTRUCTURE ONLY. The kernels take device pointers (the caller runs nsb_inference between them, standing in for tiny-cuda-nn's
// Network::inference); the writers are host code, compiled by the host compiler without FMA contraction like the reference's, and their
// stbi_write_png calls and logged counts are recorded by the stand-ins in oracle/ref_shim_slices.
#include <tiny-cuda-nn/common.h>
#include <tiny-cuda-nn/gpu_memory.h>
#include <tinylogger/tinylogger.h>

#include <atomic>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include <neural-graphics-primitives/common.h>
#include <neural-graphics-primitives/common_device.cuh>
#include <neural-graphics-primitives/common_nerf.h>
#include <neural-graphics-primitives/bounding_box.cuh>
#include <neural-graphics-primitives/nerf.h>
#include <neural-graphics-primitives/thread_pool.h>

#include <common_nerf.cu>  // /root/reference/src/common_nerf.cu, whole file

#include <stb_image/stb_image_write.h>  // oracle/ref_shim_slices
#include <thread_pool.inl>

NGP_NAMESPACE_BEGIN
using namespace Eigen;
using namespace tcnn;
#include "marching_cubes_slices.inc"
#include "testbed_nerf_slices.inc"
NGP_NAMESPACE_END

using namespace ngp;

namespace {
BoundingBox box(const float* a) { return BoundingBox{Eigen::Vector3f{a[0], a[1], a[2]}, Eigen::Vector3f{a[3], a[4], a[5]}}; }
template <typename F> int guarded(F f) {
	try {
		f();
		CUDA_CHECK_THROW(cudaGetLastError());
		return 0;
	} catch (const std::exception& e) {
		fprintf(stderr, "ref slices: %s\n", e.what());
		return 1;
	}
}
template <typename T> tcnn::GPUMemory<T> up(const void* h, size_t n) {
	tcnn::GPUMemory<T> m(n);
	if (n) CUDA_CHECK_THROW(cudaMemcpy(m.data(), h, n * sizeof(T), cudaMemcpyHostToDevice));
	return m;
}
}  // namespace

extern "C" {
uint32_t ref_slices_coordinate_floats() { return sizeof(NerfCoordinate) / sizeof(float); }

// generate_grid_samples_nerf_uniform_dir with Testbed::get_rgba_on_grid's launch (testbed_nerf.cu:4594-4597): NerfCoordinate rows into
// coords_dev (DEVICE, res[0]*res[1]*res[2] rows). Stream-ordered.
int ref_slices_grid_coords(const int32_t* res, const float* render_aabb, const float* train_aabb, const float* ray_dir, float* coords_dev, void* stream) {
	return guarded([&] {
		const Eigen::Vector3i r{res[0], res[1], res[2]};
		const dim3 threads = {16, 8, 1};
		const dim3 blocks = {div_round_up((uint32_t)r.x(), threads.x), div_round_up((uint32_t)r.y(), threads.y), div_round_up((uint32_t)r.z(), threads.z)};
		generate_grid_samples_nerf_uniform_dir<<<blocks, threads, 0, (cudaStream_t)stream>>>(r, 0u, box(render_aabb), box(train_aabb),
		                                                                                   Eigen::Vector3f{ray_dir[0], ray_dir[1], ray_dir[2]}, (NerfCoordinate*)coords_dev);
	});
}
// compute_nerf_density in place on n float4 rows (DEVICE): the network's rows 0-3 as float in, premultiplied rgba out. Stream-ordered.
int ref_slices_compute_nerf_density(uint32_t n, float* rgba_dev, int32_t rgb_activation, int32_t density_activation, void* stream) {
	return guarded([&] {
		linear_kernel(compute_nerf_density, 0, (cudaStream_t)stream, n, (Array4f*)rgba_dev, (ENerfActivation)rgb_activation, (ENerfActivation)density_activation);
	});
}
// save_density_grid_to_png on a HOST copy of the grid (uploaded first, as the reference's GPUMemory holds it)
int ref_slices_density_png(const float* density, const int32_t* res, float thresh, int32_t swap_y_z, float density_range, const char* filename) {
	return guarded([&] {
		auto d = up<float>(density, (size_t)res[0] * res[1] * res[2]);
		save_density_grid_to_png(d, filename, Eigen::Vector3i{res[0], res[1], res[2]}, thresh, swap_y_z != 0, density_range);
	});
}
// save_rgba_grid_to_png_sequence on a HOST copy of the float4 grid
int ref_slices_rgba_png(const float* rgba, const int32_t* res, int32_t swap_y_z, const char* path) {
	return guarded([&] {
		auto d = up<Array4f>(rgba, (size_t)res[0] * res[1] * res[2]);
		save_rgba_grid_to_png_sequence(d, path, Eigen::Vector3i{res[0], res[1], res[2]}, swap_y_z != 0);
	});
}
// the recorded stbi_write_png calls, in call order, and the text logged through tlog::info()
uint32_t ref_slices_n_records() { return (uint32_t)stb_png_records().size(); }
int ref_slices_record(uint32_t i, char* name, uint32_t name_capacity, int32_t* whc, uint8_t* pixels) {
	if (i >= stb_png_records().size()) return 1;
	const StbPngRecord& r = stb_png_records()[i];
	snprintf(name, name_capacity, "%s", r.filename.c_str());
	whc[0] = r.w; whc[1] = r.h; whc[2] = r.comp;
	if (pixels) std::memcpy(pixels, r.pixels.data(), r.pixels.size());
	return 0;
}
const char* ref_slices_info_text() { return tlog::info_text().c_str(); }
void ref_slices_clear() {
	stb_png_records().clear();
	tlog::info_text().clear();
}
}
