// Video frames on the device: the kernel behind nsb_frame_to_rgba8.
// Included by nsb_kernels.cu after nsb_slices.cuh (mul, add, sub, div_, clampf from nsb_device.cuh).
//
//   k_rgba8   scripts/run.py's np.clip(frame * 2**exposure, 0, 1) and write_image (scripts/common.py:122-178) for a PNG or JPEG:
//             unmultiply alpha, linear_to_srgb (:141-143), clip and quantise to 8 bits
//
// Every product and sum is rounded on its own (no contraction), as numpy evaluates the float32 arrays. powf is CUDA's, not the host
// libm's, so a byte may differ by one where the float lies within an ulp of a quantisation boundary. NaN becomes 0 (numpy leaves the
// cast of NaN to uint8 undefined; x86 gives 0).
namespace video {

// common.py's linear_to_srgb on one float32: x > 0.0031308 takes the power branch (the limit itself takes 12.92 * x)
__device__ __forceinline__ float write_image_srgb(float x) {
	return x > 0.0031308f ? sub(mul(1.055f, powf(x, (float)(1.0 / 2.4))), 0.055f) : mul(12.92f, x);
}

// (np.clip(x, 0, 1) * 255 + 0.5).astype(np.uint8)
__device__ __forceinline__ uint32_t quantise8(float x) {
	return __float2uint_rz(add(mul(clampf(x, 0.0f, 1.0f), 255.0f), 0.5f));  // NaN -> 0
}

// rgba: float4[n] linear, premultiplied (nsb_tonemap's output with a linear output colour space); scale = 2^exposure in float32.
// n_channels 4: one uchar4 per pixel (out 4-byte aligned); 3: the same RGB without alpha, three byte stores per pixel.
__global__ void k_rgba8(uint32_t n, const float4* __restrict__ rgba, float scale, int n_channels, uint8_t* __restrict__ out) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const float4 v = rgba[i];
	const float a = clampf(mul(v.w, scale), 0.0f, 1.0f);
	float c[3] = {v.x, v.y, v.z};
#pragma unroll
	for (int k = 0; k < 3; ++k) {
		const float x = clampf(mul(c[k], scale), 0.0f, 1.0f);
		c[k] = write_image_srgb(a != 0.0f ? div_(x, a) : 0.0f);
	}
	if (n_channels == 4) {
		reinterpret_cast<uchar4*>(out)[i] = make_uchar4((unsigned char)quantise8(c[0]), (unsigned char)quantise8(c[1]), (unsigned char)quantise8(c[2]),
		                                                (unsigned char)quantise8(a));
	} else {
		uint8_t* p = out + (size_t)i * 3;
		p[0] = (uint8_t)quantise8(c[0]);
		p[1] = (uint8_t)quantise8(c[1]);
		p[2] = (uint8_t)quantise8(c[2]);
	}
}

}  // namespace video
