// ref_video_driver_cuda.cu — the reference's render_frame sequence per sub-frame of Testbed::render_to_cpu (python_api.cu:129-175):
// render_buffer.clear_frame, Testbed::render_nerf, CudaRenderBuffer::accumulate (accumulate_kernel) and CudaRenderBuffer::tonemap
// (tonemap_kernel into a CUDA surface), all the reference's own code, compiled by nvcc for sm_90a into
// oracle/_ref/libnerfshop_ref_video_cuda.so by oracle/ref_video_build.py. render_to_cpu itself is pybind code and is not compiled; this
// file runs its render_frame calls on the cameras the caller gives.
// TEST INFRASTRUCTURE ONLY. The whole of oracle/ref_driver_cuda.cu (scene, render_nerf, the cut-out kernels) is included as it is.
#include "ref_driver_cuda.cu"

// render_buffer.cu's accumulate_kernel, the two tonemap() device functions and tonemap_kernel (ref_build.EXTRACTS "render_buffer"),
// which ref_common.inl compiles for the CPU build only: here they run on the GPU and write a real CUDA surface
NGP_NAMESPACE_BEGIN
using namespace Eigen;
using namespace tcnn;
#include "render_buffer.inc"
NGP_NAMESPACE_END

extern "C" {

// frames[i]: the NsbFrame render_nerf gets for sub-frame i (its spp_index is render_buffer.spp(), the accumulate's sample count).
// Every sub-frame clears fb/depth, renders, accumulates and tonemaps (render_frame, testbed.cu:2632-2765); out_dev receives the surface
// after the last one (the cudaMemcpy2DFromArray of render_to_cpu). Tonemap arguments as CudaRenderBuffer::tonemap passes them.
int refvid_render_to_cpu(void* scene, const NsbFrame* frames, int n, void* inference_fn, void* inference_ctx, float exposure, const float* background,
                         int color_space, int output_color_space, int curve, int clamp_output, float* fb_dev, float* depth_dev, float* acc_dev,
                         float* out_dev) {
	try {
		const int W = frames[0].width, H = frames[0].height;
		cudaChannelFormatDesc fmt = cudaCreateChannelDesc<float4>();
		cudaArray_t arr = nullptr;
		CUDA_CHECK_THROW(cudaMallocArray(&arr, &fmt, W, H, cudaArraySurfaceLoadStore));
		cudaResourceDesc rd{};
		rd.resType = cudaResourceTypeArray;
		rd.res.array.array = arr;
		cudaSurfaceObject_t surf = 0;
		CUDA_CHECK_THROW(cudaCreateSurfaceObject(&surf, &rd));
		const dim3 threads = {16, 8, 1};
		const dim3 blocks = {(unsigned)((W + 15) / 16), (unsigned)((H + 7) / 8), 1};
		uint64_t stats[3];
		for (int i = 0; i < n; ++i) {
			CUDA_CHECK_THROW(cudaMemset(fb_dev, 0, (size_t)W * H * 16));
			CUDA_CHECK_THROW(cudaMemset(depth_dev, 0, (size_t)W * H * 4));
			if (refcu_render(scene, &frames[i], inference_fn, inference_ctx, fb_dev, depth_dev, nullptr, stats) != 0) throw std::runtime_error("refcu_render failed");
			const uint32_t spp = frames[i].spp_index;
			if (spp == 0) CUDA_CHECK_THROW(cudaMemset(acc_dev, 0, (size_t)W * H * 16));
			accumulate_kernel<<<blocks, threads>>>(Vector2i(W, H), (Array4f*)fb_dev, (Array4f*)acc_dev, (float)spp, (EColorSpace)color_space);
			tonemap_kernel<<<blocks, threads>>>(Vector2i(W, H), exposure, Array4f(background[0], background[1], background[2], background[3]), (Array4f*)acc_dev,
			                                    (EColorSpace)color_space, (EColorSpace)output_color_space, (ETonemapCurve)curve, clamp_output != 0, surf, nullptr);
			CUDA_CHECK_THROW(cudaGetLastError());
		}
		CUDA_CHECK_THROW(cudaMemcpy2DFromArray(out_dev, (size_t)W * 16, arr, 0, 0, (size_t)W * 16, H, cudaMemcpyDeviceToDevice));
		CUDA_CHECK_THROW(cudaDeviceSynchronize());
		cudaDestroySurfaceObject(surf);
		cudaFreeArray(arr);
		return 0;
	} catch (const std::exception& e) {
		fprintf(stderr, "refvid_render_to_cpu: %s\n", e.what());
		return 1;
	}
}

// The post-process alone on caller buffers, as CudaRenderBuffer::accumulate and ::tonemap launch it (render_buffer.cu:540-579), 16x8
// blocks. n_frames accumulate_kernel calls, frame i (frames_dev + i*W*H*4) with sample count spp0 + i (a zeroed accumulation first when
// that is 0); acc_hist_dev, when given, receives the accumulation after every call ([n_frames][W*H][4]). Then, when out_dev is given,
// tonemap_kernel of the accumulation into a CUDA surface once per row of tm ([n_tm][9]: exposure, background rgba, output colour space,
// curve, clamp, unused), with the full argument list; out_dev[k] receives surface k ([n_tm][W*H][4], cudaMemcpy2DFromArray).
// frames_dev may be null (n_frames 0): acc_dev is then tonemapped as the caller wrote it.
int refvid_postprocess(const float* frames_dev, int n_frames, uint32_t spp0, int W, int H, int color_space, float* acc_dev, float* acc_hist_dev,
                       const float* tm, int n_tm, float* out_dev) {
	try {
		const dim3 threads = {16, 8, 1};
		const dim3 blocks = {(unsigned)((W + 15) / 16), (unsigned)((H + 7) / 8), 1};
		const size_t px = (size_t)W * H;
		for (int i = 0; i < n_frames; ++i) {
			const uint32_t spp = spp0 + (uint32_t)i;
			if (spp == 0) CUDA_CHECK_THROW(cudaMemset(acc_dev, 0, px * 16));
			accumulate_kernel<<<blocks, threads>>>(Vector2i(W, H), (Array4f*)(frames_dev + px * 4 * i), (Array4f*)acc_dev, (float)spp, (EColorSpace)color_space);
			CUDA_CHECK_THROW(cudaGetLastError());
			if (acc_hist_dev) CUDA_CHECK_THROW(cudaMemcpy(acc_hist_dev + px * 4 * i, acc_dev, px * 16, cudaMemcpyDeviceToDevice));
		}
		if (out_dev && n_tm > 0) {
			cudaChannelFormatDesc fmt = cudaCreateChannelDesc<float4>();
			cudaArray_t arr = nullptr;
			CUDA_CHECK_THROW(cudaMallocArray(&arr, &fmt, W, H, cudaArraySurfaceLoadStore));
			cudaResourceDesc rd{};
			rd.resType = cudaResourceTypeArray;
			rd.res.array.array = arr;
			cudaSurfaceObject_t surf = 0;
			CUDA_CHECK_THROW(cudaCreateSurfaceObject(&surf, &rd));
			for (int k = 0; k < n_tm; ++k) {
				const float* t = tm + 9 * (size_t)k;
				tonemap_kernel<<<blocks, threads>>>(Vector2i(W, H), t[0], Array4f(t[1], t[2], t[3], t[4]), (Array4f*)acc_dev, (EColorSpace)color_space,
				                                    (EColorSpace)(int)t[5], (ETonemapCurve)(int)t[6], t[7] != 0.0f, surf, nullptr);
				CUDA_CHECK_THROW(cudaGetLastError());
				CUDA_CHECK_THROW(cudaMemcpy2DFromArray(out_dev + px * 4 * k, (size_t)W * 16, arr, 0, 0, (size_t)W * 16, H, cudaMemcpyDeviceToDevice));
			}
			CUDA_CHECK_THROW(cudaDeviceSynchronize());
			cudaDestroySurfaceObject(surf);
			cudaFreeArray(arr);
		}
		CUDA_CHECK_THROW(cudaDeviceSynchronize());
		return 0;
	} catch (const std::exception& e) {
		fprintf(stderr, "refvid_postprocess: %s\n", e.what());
		return 1;
	}
}

}  // extern "C"
