// Image-quality metrics on the device: the kernels behind nsb_reference_image and nsb_image_metrics.
// Included by nsb_kernels.cu after nsb_video.cuh. It uses CUDA intrinsics only, so a test can compile its device functions on their own.
//
//   k_reference_image  scripts/common.py's read_image (:147-161) on decoded 8-bit pixels, and run.py's sRGB blend (run.py:264-270)
//   k_image_metrics    run.py's per-frame block (run.py:286-290): A and R, then compute_error("MSE") and compute_error("SSIM")
//                      (common.py:190-207, 227-275) up to their two float32 maps
//   k_pairwise_nodes,  np.mean of each map: numpy's pairwise float32 sum (numpy/_core/src/umath/loops_utils.h.src) evaluated as the
//   k_pairwise_root    fixed tree it builds for n elements, then float32(float64(sum) / n)
//
// numpy evaluates every step in float32 with each operation rounded on its own, so every product, sum and quotient below is an _rn
// intrinsic (no contraction), in numpy's operation order. The one exception is pow: numpy's float32 `**` depends on the host (on AVX-512
// it dispatches to SIMD code that is not correctly rounded, elsewhere to libm), so pow here is the float64 pow, rounded once to float32.
// That is the correctly rounded result except where the exact power lies closer to a float32 rounding boundary than float64 pow's own
// error: one float32 in [0, 1] for the luminance exponent, none for the other two (DESIGN §7.6). Constants are Python doubles rounded
// to float32, as numpy's weak scalars are.
namespace evalm {

__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float div_(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float pow_cr(float x, float y) { return __double2float_rn(pow((double)x, (double)y)); }

// np.clip(x, 0, 1) on float32: NaN kept, and -0 kept as numpy's clip keeps it
__device__ __forceinline__ float clip01(float x) {
	if (x != x) return x;
	const float m = x >= 0.0f ? x : 0.0f;
	return m <= 1.0f ? m : 1.0f;
}

// common.py:139-145
__device__ __forceinline__ float srgb_to_linear(float x) {
	return x > (float)0.04045 ? pow_cr(div_(add(x, (float)0.055), (float)1.055), (float)2.4) : div_(x, (float)12.92);
}
__device__ __forceinline__ float linear_to_srgb(float x) {
	return x > (float)0.0031308 ? sub(mul((float)1.055, pow_cr(x, (float)(1.0 / 2.4))), (float)0.055) : mul((float)12.92, x);
}

// luminance's np.maximum(0, a) ** 0.4545454545 (common.py:186-188) for one channel: 0 >= a gives 0, NaN stays
__device__ __forceinline__ float lum_pow(float a) { return pow_cr(0.0f >= a ? 0.0f : a, (float)0.4545454545); }
__device__ __forceinline__ float luminance(float p0, float p1, float p2) {
	return add(add(mul((float)0.2126, p0), mul((float)0.7152, p1)), mul((float)0.0722, p2));
}

// A for one channel of the rendered frame: np.clip(linear_to_srgb(x), 0, 1), then compute_error_img's clean-up (non-finite -> 0,
// np.maximum(., 0)); R is the same without the clean-up
__device__ __forceinline__ float metric_a(float x) {
	const float a = clip01(linear_to_srgb(x));
	return isfinite(a) && a > 0.0f ? a : 0.0f;
}
__device__ __forceinline__ float metric_r(float x) { return clip01(linear_to_srgb(x)); }

// compute_error("MSE") per pixel: L2 per channel, non-finite -> 0, np.mean(axis=2) = float32(float64((s0 + s1) + s2) / 3)
__device__ __forceinline__ float mse_pixel(const float a[3], const float r[3]) {
	float s[3];
#pragma unroll
	for (int k = 0; k < 3; ++k) {
		const float d = sub(a[k], r[k]);
		s[k] = mul(d, d);
		if (!isfinite(s[k])) s[k] = 0.0f;
	}
	return __double2float_rn(__ddiv_rn((double)add(add(s[0], s[1]), s[2]), 3.0));
}

// SSIM's luminance of A and R (their np.clip(., 0, 1) is the identity on A; it keeps R's NaN)
__device__ __forceinline__ float lum_of(const float c[3]) { return luminance(lum_pow(clip01(c[0])), lum_pow(clip01(c[1])), lum_pow(clip01(c[2]))); }

// scipy.ndimage's 'reflect' boundary (np.pad mode "symmetric") for any index, including lines shorter than the 2-pixel halo
__device__ __forceinline__ int reflect(int i, int n) {
	while (i < 0 || i >= n) i = i < 0 ? -i - 1 : 2 * n - 1 - i;
	return i;
}

// convolve1d's symmetric-kernel loop (scipy/ndimage/src/ni_filters.c, NI_Correlate1D) in float64 on float32 samples x[-2..2]:
// x0 * k2, then + (x-2 + x2) * k0, then + (x-1 + x1) * k1, rounded once to float32
__device__ __forceinline__ float blur5(float m2, float m1, float c, float p1, float p2) {
	double t = __dmul_rn((double)c, 0.292082);
	t = __dadd_rn(t, __dmul_rn(__dadd_rn((double)m2, (double)p2), 0.120078));
	t = __dadd_rn(t, __dmul_rn(__dadd_rn((double)m1, (double)p1), 0.233881));
	return __double2float_rn(t);
}

// common.py:200-207 on the five blurred maps: p1 * p2, non-finite -> 0 (compute_error)
__device__ __forceinline__ float ssim_pixel(float mA, float mB, float bAA, float bBB, float bAB) {
	const float c1 = (float)(0.01 * 0.01), c2 = (float)(0.03 * 0.03);
	const float sA = sub(bAA, mul(mA, mA)), sB = sub(bBB, mul(mB, mB)), sAB = sub(bAB, mul(mA, mB));
	const float p1 = div_(add(mul(mul(2.0f, mA), mB), c1), add(add(mul(mA, mA), mul(mB, mB)), c1));
	const float p2 = div_(add(mul(2.0f, sAB), c2), add(add(sA, sB), c2));
	const float e = mul(p1, p2);
	return isfinite(e) ? e : 0.0f;
}

// ---- ground truth --------------------------------------------------------------------------------------------------
// read_image on 8-bit pixels: byte / 255, srgb_to_linear on the colour, colour * alpha (RGB: alpha 1). srgb_blend (RGBA only): run.py's
// NeRF-compatible blend: unmultiply, linear_to_srgb, re-multiply, + (1 - alpha) * background on all four channels, srgb_to_linear.
__global__ void k_reference_image(uint32_t n, const uint8_t* __restrict__ px, int n_channels, int srgb_blend, float4 bg, float4* __restrict__ out) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const uint8_t* p = px + (size_t)i * n_channels;
	float c[3];
#pragma unroll
	for (int k = 0; k < 3; ++k) c[k] = srgb_to_linear(div_((float)p[k], 255.0f));
	if (n_channels == 3) {
		out[i] = make_float4(c[0], c[1], c[2], 1.0f);
		return;
	}
	float a = div_((float)p[3], 255.0f);
#pragma unroll
	for (int k = 0; k < 3; ++k) c[k] = mul(c[k], a);
	if (srgb_blend) {
		const float t = sub(1.0f, a), b[3] = {bg.x, bg.y, bg.z};
#pragma unroll
		for (int k = 0; k < 3; ++k) {
			const float u = a != 0.0f ? div_(c[k], a) : 0.0f;
			c[k] = srgb_to_linear(add(mul(linear_to_srgb(u), a), mul(t, b[k])));
		}
		a = add(a, mul(t, bg.w));
	}
	out[i] = make_float4(c[0], c[1], c[2], a);
}

// ---- the two maps --------------------------------------------------------------------------------------------------
// One TX x TY tile of output pixels per CTA. The luminances of A and R are computed once per tile pixel and halo pixel (2 on each side,
// reflected), the five maps a, b, a*a, b*b, a*b are blurred along axis 0 into shared memory and then along axis 1, as convolve1d does.
constexpr int kTX = 32, kTY = 16, kHalo = 2, kSX = kTX + 2 * kHalo, kSY = kTY + 2 * kHalo;
constexpr int kThreads = 256;

__global__ void __launch_bounds__(kThreads) k_image_metrics(int W, int H, const float4* __restrict__ image, const float4* __restrict__ ref,
                                                            float* __restrict__ mse_map, float* __restrict__ ssim_map) {
	__shared__ float la[kSY][kSX], lb[kSY][kSX];
	__shared__ float vb[5][kTY][kSX];  // axis-0 blur of a, b, a*a, b*b, a*b
	const int x0 = blockIdx.x * kTX, y0 = blockIdx.y * kTY, tid = threadIdx.x;
	for (int s = tid; s < kSY * kSX; s += kThreads) {
		const int sy = s / kSX, sx = s % kSX, gy = y0 + sy - kHalo, gx = x0 + sx - kHalo;
		const size_t p = (size_t)reflect(gy, H) * W + reflect(gx, W);
		const float4 v = image[p], w = ref[p];
		const float A[3] = {metric_a(v.x), metric_a(v.y), metric_a(v.z)};
		const float R[3] = {metric_r(w.x), metric_r(w.y), metric_r(w.z)};
		la[sy][sx] = lum_of(A);
		lb[sy][sx] = lum_of(R);
		if (sy >= kHalo && sy < kHalo + kTY && sx >= kHalo && sx < kHalo + kTX && gy < H && gx < W) mse_map[p] = mse_pixel(A, R);
	}
	__syncthreads();
	for (int s = tid; s < kTY * kSX; s += kThreads) {
		const int ty = s / kSX, sx = s % kSX;
		float a[5], b[5];
#pragma unroll
		for (int k = 0; k < 5; ++k) a[k] = la[ty + k][sx], b[k] = lb[ty + k][sx];
		vb[0][ty][sx] = blur5(a[0], a[1], a[2], a[3], a[4]);
		vb[1][ty][sx] = blur5(b[0], b[1], b[2], b[3], b[4]);
		vb[2][ty][sx] = blur5(mul(a[0], a[0]), mul(a[1], a[1]), mul(a[2], a[2]), mul(a[3], a[3]), mul(a[4], a[4]));
		vb[3][ty][sx] = blur5(mul(b[0], b[0]), mul(b[1], b[1]), mul(b[2], b[2]), mul(b[3], b[3]), mul(b[4], b[4]));
		vb[4][ty][sx] = blur5(mul(a[0], b[0]), mul(a[1], b[1]), mul(a[2], b[2]), mul(a[3], b[3]), mul(a[4], b[4]));
	}
	__syncthreads();
	for (int s = tid; s < kTY * kTX; s += kThreads) {
		const int ty = s / kTX, tx = s % kTX, gy = y0 + ty, gx = x0 + tx;
		if (gy >= H || gx >= W) continue;
		float m[5];
#pragma unroll
		for (int k = 0; k < 5; ++k) m[k] = blur5(vb[k][ty][tx], vb[k][ty][tx + 1], vb[k][ty][tx + 2], vb[k][ty][tx + 3], vb[k][ty][tx + 4]);
		ssim_map[(size_t)gy * W + gx] = ssim_pixel(m[0], m[1], m[2], m[3], m[4]);
	}
}

// ---- np.mean of a float32 map ----------------------------------------------------------------------------------------
// numpy's pairwise_sum: n < 8 summed in order from -0.0; n <= 128 in eight strided accumulators combined ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7))
// plus the tail in order; larger n split at n/2 rounded down to a multiple of 8. The tree depends on n only, so it is evaluated as a fixed
// tree: k_pairwise_nodes sums the subtrees at depth kDepth (one thread each), k_pairwise_root adds them up level by level.
constexpr int kDepth = 14;
constexpr uint32_t kLeaf = 128;

__device__ __forceinline__ uint32_t split(uint32_t n) { const uint32_t h = n / 2; return h - h % 8; }

__device__ float pairwise_leaf(const float* a, uint32_t n) {
	if (n < 8) {
		float r = -0.0f;
		for (uint32_t i = 0; i < n; ++i) r = add(r, a[i]);
		return r;
	}
	float r[8];
#pragma unroll
	for (int j = 0; j < 8; ++j) r[j] = a[j];
	uint32_t i = 8;
	for (; i < n - n % 8; i += 8) {
#pragma unroll
		for (int j = 0; j < 8; ++j) r[j] = add(r[j], a[i + j]);
	}
	float res = add(add(add(r[0], r[1]), add(r[2], r[3])), add(add(r[4], r[5]), add(r[6], r[7])));
	for (; i < n; ++i) res = add(res, a[i]);
	return res;
}

// the whole recursion for one subtree, with an explicit stack (every split at least halves n, so 32 levels cover 2^32 elements)
__device__ float pairwise_sum(const float* a, uint32_t n) {
	uint32_t r_off[32], r_n[32];
	float left[32];
	bool on_right[32];
	int sp = 0;
	uint32_t off = 0;
	for (;;) {
		while (n > kLeaf) {
			const uint32_t n2 = split(n);
			r_off[sp] = off + n2, r_n[sp] = n - n2, on_right[sp] = false;
			++sp;
			n = n2;
		}
		float v = pairwise_leaf(a + off, n);
		for (;;) {
			if (sp == 0) return v;
			if (!on_right[sp - 1]) {
				left[sp - 1] = v, on_right[sp - 1] = true, off = r_off[sp - 1], n = r_n[sp - 1];
				break;
			}
			--sp;
			v = add(left[sp], v);
		}
	}
}

// Node t at depth d of the tree over n elements (t's d bits, most significant first: 0 left, 1 right). A leaf above depth d is carried by
// its leftmost descendant; every other descendant of it is empty (false).
__device__ __forceinline__ bool tree_node(uint32_t n, int d, uint32_t t, uint32_t& off, uint32_t& len) {
	off = 0, len = n;
	for (int k = d - 1; k >= 0; --k) {
		const bool right = (t >> k) & 1u;
		if (len > kLeaf) {
			const uint32_t n2 = split(len);
			if (right) off += n2, len -= n2;
			else len = n2;
		} else if (right) {
			return false;
		}
	}
	return true;
}

// heap: per map, 2^(kDepth+1) floats; depth d's nodes at [2^d, 2^(d+1)). blockIdx.y: the map.
__global__ void k_pairwise_nodes(uint32_t n, const float* __restrict__ map0, const float* __restrict__ map1, float* __restrict__ heap) {
	const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= (1u << kDepth)) return;
	const float* map = blockIdx.y ? map1 : map0;
	uint32_t off, len;
	heap[(size_t)blockIdx.y * (2u << kDepth) + (1u << kDepth) + t] = tree_node(n, kDepth, t, off, len) ? pairwise_sum(map + off, len) : 0.0f;
}

// one CTA per map: the levels above kDepth, then np.mean's float32(float64(sum) / n) into out[blockIdx.x]
__global__ void __launch_bounds__(1024) k_pairwise_root(uint32_t n, float* __restrict__ heap, float* __restrict__ out) {
	float* h = heap + (size_t)blockIdx.x * (2u << kDepth);
	for (int d = kDepth - 1; d >= 0; --d) {
		for (uint32_t p = threadIdx.x; p < (1u << d); p += blockDim.x) {
			uint32_t off, len;
			if (!tree_node(n, d, p, off, len)) continue;
			const float* c = h + (2u << d) + 2 * p;
			h[(1u << d) + p] = len > kLeaf ? add(c[0], c[1]) : c[0];
		}
		__syncthreads();
	}
	if (threadIdx.x == 0) out[blockIdx.x] = __double2float_rn(__ddiv_rn((double)h[1], (double)n));
}

}  // namespace evalm
