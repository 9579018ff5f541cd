// nsb_tc.cuh — Hopper warpgroup tensor core (wgmma) plumbing for the fully fused 64-wide MLPs.
//
// Geometry: one tile = 128 threads = one warpgroup = 128 samples; thread t owns sample t and (in the fused renderer) ray t.
// The five layers
//     L1 32->64 (ReLU)  L2 64->16        (density MLP, base.json "network")
//     L3 32->64 (ReLU)  L4 64->64 (ReLU)  L5 64->16   (rgb MLP, "rgb_network")
// run as wgmma.mma_async m64nNk16 (K=16 per instruction), one M=64 half of the tile at a time, accumulators in registers.
// L1 and L3 read their A operand from shared memory (written row by row by the threads that own the samples); L2, L4 and L5
// take it straight from the previous layer's accumulators (the m64nNk16 accumulator fragment is the A fragment of the next
// layer), so hidden activations never leave the registers. The weights (20 KB) are staged once per CTA by a bulk-TMA copy.
//
// Shared-memory operand layout (K-major, no swizzle = the wgmma "interleave" canonical layout
// ((8,m),(T,2)):((1T,SBO),(1,LBO)) in 16-byte units):
//   element (physical row p, k) of an [R x K] fp16 operand lives at  (k/8)*(R*16) + p*16 + (k%8)*2  bytes
//   -> core matrix = 8 rows x 16 B contiguous (128 B); SBO (next 8 rows) = 128 B; LBO (next 8 k) = R*16 B.
// Row permutation: warp w of a warpgroup receives accumulator rows 16w..16w+15 of each M=64 half. Sample t is stored at physical
// row phys_row(t) = 64*((t%32)/16) + 16*(t/32) + t%16, so every accumulator row a warp receives belongs to one of its own 32
// threads: the result hand-back to the owning thread is a warp-local exchange through the warp's own operand rows.
#pragma once

#include <cuda_fp16.h>
#include <stdint.h>

#include "nsb_device.cuh"

namespace nsb {
namespace tc {

constexpr uint32_t ROWS = 128;                    // samples per tile = one warpgroup, two M=64 halves
constexpr uint32_t A32_BYTES = 4 * ROWS * 16;     // [4 k-chunks][128][16 B]
constexpr uint32_t A64_BYTES = 8 * ROWS * 16;
// weight image: W1 [64x32], W2 [16x64], W3 [64x32], W4 [64x64], W5 [16x64], each in the operand layout above
constexpr uint32_t W1_OFF = 0;
constexpr uint32_t W2_OFF = W1_OFF + 64 * 32 * 2;
constexpr uint32_t W3_OFF = W2_OFF + 16 * 64 * 2;
constexpr uint32_t W4_OFF = W3_OFF + 64 * 32 * 2;
constexpr uint32_t W5_OFF = W4_OFF + 64 * 64 * 2;
constexpr uint32_t W_BYTES = W5_OFF + 16 * 64 * 2;  // 20480

// Operand space of a tile: chunks 0-3 = the 32-wide layer input (grid features for L1; density output + SH for L3), chunks 4-5 =
// the hand-back of the rgb output. The a32 view aliases the first half of a64.
struct __align__(128) TileSmem {
	uint8_t w[W_BYTES];
	union {
		uint8_t a64[A64_BYTES];
		uint8_t a32[A32_BYTES];
	};
	uint64_t w_bar;
	uint32_t pad[2];
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__host__ __device__ __forceinline__ uint32_t phys_row(uint32_t t) { return ((t & 16u) << 2) | ((t >> 5) << 4) | (t & 15u); }

// ---- mbarrier -----------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
	asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// Bounded wait: a broken pipeline traps (after ~2 s) instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
	uint32_t addr = smem_u32(bar);
	uint32_t done = 0;
	long long t0 = 0;
	for (uint32_t spins = 0; !done; ++spins) {
		asm volatile(
			"{\n\t.reg .pred p;\n\t"
			"mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
			"selp.u32 %0, 1, 0, p;\n\t}"
			: "=r"(done)
			: "r"(addr), "r"(parity)
			: "memory");
		if (!done && (spins & 1023u) == 1023u) {
			long long now = clock64();
			if (t0 == 0) t0 = now;
			else if (now - t0 > 4000000000ll) __trap();
		}
	}
}
// The same wait for a barrier whose completion is thousands of cycles away (the warp-specialised renderer's producer <-> consumer hand-offs):
// a spinning warp takes issue slots from the warps it is waiting for, so back off with nanosleep between polls.
__device__ __forceinline__ void mbar_wait_backoff(uint64_t* bar, uint32_t parity, uint32_t ns) {
	uint32_t addr = smem_u32(bar);
	uint32_t done = 0;
	long long t0 = 0;
	for (uint32_t spins = 0;; ++spins) {
		asm volatile(
			"{\n\t.reg .pred p;\n\t"
			"mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
			"selp.u32 %0, 1, 0, p;\n\t}"
			: "=r"(done)
			: "r"(addr), "r"(parity)
			: "memory");
		if (done) break;
		__nanosleep(ns);
		if ((spins & 4095u) == 4095u) {
			long long now = clock64();
			if (t0 == 0) t0 = now;
			else if (now - t0 > 8000000000ll) __trap();
		}
	}
}
// bulk TMA copy global -> shared, completion on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src),
	             "r"(bytes), "r"(smem_u32(bar))
	             : "memory");
}
// generic-proxy shared stores -> visible to the async proxy (tensor core operand reads)
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// One thread stages the weight image (bulk TMA) and initialises the barrier; the caller's __syncthreads() publishes the init,
// then every thread waits for the copy.
__device__ __forceinline__ void load_weights(uint8_t* w, uint64_t* w_bar, const uint8_t* __restrict__ w_image) {
	if (threadIdx.x == 0) {
		mbar_init(w_bar, 1);
		fence_mbar_init();
		mbar_expect_tx(w_bar, W_BYTES);
		bulk_g2s(w, w_image, W_BYTES, w_bar);
	}
}

// ---- wgmma ------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor (sm_90 GMMA): start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46), base_offset [49,52)=0,
// layout_type [62,64)=0 (INTERLEAVE, no swizzle).
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
	uint64_t d = 0;
	d |= (uint64_t)((smem_addr >> 4) & 0x3fffu);
	d |= (uint64_t)((lbo_bytes >> 4) & 0x3fffu) << 16;
	d |= (uint64_t)((sbo_bytes >> 4) & 0x3fffu) << 32;
	return d;
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMA
template <int NR> __device__ __forceinline__ void reg_fence(uint32_t* r) {
#pragma unroll
	for (int i = 0; i < NR; ++i) asm volatile("" : "+r"(r[i])::"memory");
}

// Accumulators per thread of one m64nNk16: N/2 fp32 (ACC16 = false) or N/4 packed half2 (ACC16 = true), as 32-bit registers.
// acc16: D=F16 — the accumulator is rounded to fp16 by every K=16 instruction, the arithmetic of wmma m16n16k16 with __half
// accumulator fragments (tiny-cuda-nn's FullyFusedMLP of the reference's era).
template <uint32_t N, bool ACC16> struct Acc { static constexpr int R = ACC16 ? (int)N / 4 : (int)N / 2; uint32_t r[R] = {}; };

// D[64 x N] (+)= A[64 x 16] * B[N x 16]^T. _ss: A from shared memory (descriptor); _rs: A from registers (4 x half2 fragment).
// B is the weight operand in shared memory; scale_d = 0 overwrites D. Both operands K-major (no transpose).
template <uint32_t N, bool ACC16> __device__ __forceinline__ void wgmma_ss(uint32_t* d, uint64_t ad, uint64_t bd, uint32_t scale_d);
template <uint32_t N, bool ACC16> __device__ __forceinline__ void wgmma_rs(uint32_t* d, const uint32_t* a, uint64_t bd, uint32_t scale_d);
template <> __device__ __forceinline__ void wgmma_ss<64, false>(uint32_t* d, uint64_t ad, uint64_t bd, uint32_t scale_d) {
	asm volatile(
		"{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
		"wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
		"{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
		: "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
		: "l"(ad), "l"(bd), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_ss<64, true>(uint32_t* d, uint64_t ad, uint64_t bd, uint32_t scale_d) {
	asm volatile(
		"{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
		"wgmma.mma_async.sync.aligned.m64n64k16.f16.f16.f16 "
		"{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
		: "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
		: "l"(ad), "l"(bd), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_rs<64, false>(uint32_t* d, const uint32_t* a, uint64_t bd, uint32_t scale_d) {
	asm volatile(
		"{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
		"wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
		"{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
		: "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
		: "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bd), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_rs<64, true>(uint32_t* d, const uint32_t* a, uint64_t bd, uint32_t scale_d) {
	asm volatile(
		"{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
		"wgmma.mma_async.sync.aligned.m64n64k16.f16.f16.f16 "
		"{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}"
		: "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
		: "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bd), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_rs<16, false>(uint32_t* d, const uint32_t* a, uint64_t bd, uint32_t scale_d) {
	asm volatile(
		"{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
		"wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
		"{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, 0;\n\t}"
		: "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7])
		: "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bd), "r"(scale_d));
}
template <> __device__ __forceinline__ void wgmma_rs<16, true>(uint32_t* d, const uint32_t* a, uint64_t bd, uint32_t scale_d) {
	asm volatile(
		"{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %9, 0;\n\t"
		"wgmma.mma_async.sync.aligned.m64n16k16.f16.f16.f16 "
		"{%0, %1, %2, %3}, {%4, %5, %6, %7}, %8, p, 1, 1, 0;\n\t}"
		: "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
		: "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bd), "r"(scale_d));
}

// ---- fragments --------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_h2(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }
__device__ __forceinline__ uint32_t pack(uint32_t a_bits, uint32_t b_bits) {
	return pack_h2(__floats2half2_rn(__uint_as_float(a_bits), __uint_as_float(b_bits)));
}
// ReLU after the fp16 conversion: rounding is monotone and 0 is exact, so max(cvt(x), 0) == cvt(max(x, 0)) — one packed
// HMNMX2 per pair instead of two FMNMX.
__device__ __forceinline__ uint32_t relu_h2(uint32_t p) { return pack_h2(__hmax2(*reinterpret_cast<__half2*>(&p), __floats2half2_rn(0.0f, 0.0f))); }
// Element pair i of an accumulator as packed half2, in fragment order: pair i covers row (lane/4 + 8*(i&1)), columns 8*(i/2) + 2*(lane%4) + {0,1}
// of the warp's 16 rows. fp32 accumulators are rounded here, fp16 accumulators already are pairs.
template <bool ACC16> __device__ __forceinline__ uint32_t acc_pair(const uint32_t* d, int i) { return ACC16 ? d[i] : pack(d[2 * i], d[2 * i + 1]); }

// One layer on one M=64 half: D = A * W^T with A in shared memory (a_addr = the half's first row, k-chunk stride ROWS*16)
template <uint32_t N, uint32_t K, bool ACC16>
__device__ __forceinline__ void layer_ss(uint32_t* d, uint32_t a_addr, uint32_t w_addr) {
	wg_fence();
#pragma unroll
	for (uint32_t k = 0; k < K / 16; ++k)  // one instruction consumes K=16 = two 8-wide k-chunks
		wgmma_ss<N, ACC16>(d, make_desc(a_addr + k * 2 * (ROWS * 16), ROWS * 16, 128), make_desc(w_addr + k * 2 * (N * 16), N * 16, 128), k > 0 ? 1u : 0u);
	wg_commit();
	wg_wait();
	reg_fence<Acc<N, ACC16>::R>(d);
}
// ... with A = ReLU(the previous layer's accumulators `x` of width K): the accumulator fragment of columns 16k..16k+15 is the A fragment of k-step k
template <uint32_t N, uint32_t K, bool ACC16>
__device__ __forceinline__ void layer_rs(uint32_t* d, const uint32_t* x, uint32_t w_addr) {
	uint32_t a[K / 16][4];
#pragma unroll
	for (uint32_t k = 0; k < K / 16; ++k)
#pragma unroll
		for (int i = 0; i < 4; ++i) a[k][i] = relu_h2(acc_pair<ACC16>(x, 4 * (int)k + i));
	wg_fence();
#pragma unroll
	for (uint32_t k = 0; k < K / 16; ++k) wgmma_rs<N, ACC16>(d, a[k], make_desc(w_addr + k * 2 * (N * 16), N * 16, 128), k > 0 ? 1u : 0u);
	wg_commit();
	wg_wait();
	reg_fence<Acc<N, ACC16>::R>(d);
}

// ---- a tile = 128 threads (one warpgroup) walking the layer chain together. A CTA may hold several tiles
// (they share the weight image; each has its own operand space and named barrier).
struct TileCtx {
	uint8_t* a32;        // operand space (A64_BYTES); the 32-wide operand is its first half
	uint32_t w_addr;     // shared-window address of the weight image
	uint32_t row;        // sample 0..127 within the tile
	uint32_t bar_id;     // named barrier of the tile (0 = the CTA barrier when the CTA is one tile)
};
__device__ __forceinline__ void tile_sync(const TileCtx& c) { asm volatile("bar.sync %0, 128;" ::"r"(c.bar_id) : "memory"); }
__device__ __forceinline__ bool tile_any(const TileCtx& c, bool p) {
	uint32_t r;
	asm volatile(
		"{\n\t.reg .pred p, q;\n\t"
		"setp.ne.u32 q, %2, 0;\n\t"
		"barrier.cta.red.or.pred p, %1, 128, q;\n\t"
		"selp.u32 %0, 1, 0, p;\n\t}"
		: "=r"(r)
		: "r"(c.bar_id), "r"((uint32_t)p)
		: "memory");
	return r != 0;
}

// ---- tile lifecycle (one-tile CTAs) ----------------------------------------------------------------
__device__ __forceinline__ void tile_setup(TileSmem& s, const uint8_t* __restrict__ w_image) {
	load_weights(s.w, &s.w_bar, w_image);
	__syncthreads();
	mbar_wait(&s.w_bar, 0);
}
__device__ __forceinline__ TileCtx single_tile_ctx(TileSmem& s) {
	TileCtx c;
	c.a32 = s.a32; c.w_addr = smem_u32(s.w); c.row = threadIdx.x; c.bar_id = 0;
	return c;
}

// ---- operand row stores ------------------------------------------------------------------------------
// 8 consecutive fp16 (one 16-byte k-chunk) of sample `row`
__device__ __forceinline__ void store_chunk(uint8_t* base, uint32_t chunk, uint32_t row, uint4 v) {
	*reinterpret_cast<uint4*>(base + chunk * (ROWS * 16) + phys_row(row) * 16) = v;
}
__device__ __forceinline__ uint4 load_chunk(const uint8_t* base, uint32_t chunk, uint32_t row) {
	return *reinterpret_cast<const uint4*>(base + chunk * (ROWS * 16) + phys_row(row) * 16);
}
// A 16-wide output (this lane's 4 pairs of half `h`) -> k-chunks `chunk`, `chunk`+1 of the warp's own physical rows
template <bool ACC16>
__device__ __forceinline__ void store_out16(uint8_t* base, uint32_t chunk, uint32_t row, uint32_t h, const uint32_t* d) {
	const uint32_t lane = row & 31u;
	uint8_t* p = base + chunk * (ROWS * 16) + (64u * h + 16u * (row >> 5) + (lane >> 2)) * 16 + (lane & 3u) * 4;
	*reinterpret_cast<uint32_t*>(p) = acc_pair<ACC16>(d, 0);
	*reinterpret_cast<uint32_t*>(p + 8 * 16) = acc_pair<ACC16>(d, 1);
	*reinterpret_cast<uint32_t*>(p + ROWS * 16) = acc_pair<ACC16>(d, 2);
	*reinterpret_cast<uint32_t*>(p + ROWS * 16 + 8 * 16) = acc_pair<ACC16>(d, 3);
}

// Runs the network on the tile's 128 samples whose grid features are already in the first layer's operand.
//   density_only: stop after L2 (NerfNetwork::density)
//   dens[8]: the 16 fp16 outputs of the density MLP (packed half2), rgb[8]: the 16 outputs of the rgb MLP, both for sample c.row.
// `dw` = this sample's warped view direction; its 16 SH values are evaluated between L2 and L3.
// `a_first`: shared-window address of the first layer's operand when it does not live in c.a32 (the warp-specialised renderer's producers
// write the grid features into their own operand); 0 = c.a32. `release`: an mbarrier to arrive on (one arrival) once every warp's first
// layer has read that operand.
// Operand space: chunks 0-3 the 32-wide layer inputs, 4-5 the rgb hand-back, 6-7 the density hand-back. On return the whole tile has
// finished with the operand space, so the caller may overwrite any of it.
template <bool ACC16 = false>
__device__ __forceinline__ void run_network(const TileCtx& c, V3 dw, bool density_only, uint32_t* dens, uint32_t* rgb, uint32_t a_first = 0,
                                            uint64_t* release = nullptr) {
	const uint32_t row = c.row;
	const uint32_t a32 = smem_u32(c.a32), w = c.w_addr;
	if (a_first == 0) a_first = a32;
	fence_async_smem();
	tile_sync(c);  // every sample's grid features are in place
#pragma unroll 1
	for (uint32_t h = 0; h < 2; ++h) {
		Acc<64, ACC16> x;
		Acc<16, ACC16> o;
		layer_ss<64, 32, ACC16>(x.r, a_first + h * 64 * 16, w + W1_OFF);  // L1: grid features (32) -> 64
		layer_rs<16, 64, ACC16>(o.r, x.r, w + W2_OFF);                    // L2: 64 -> 16
		store_out16<ACC16>(c.a32, 6, row, h, o.r);
	}
	__syncwarp();
	{
		const uint4 d0 = load_chunk(c.a32, 6, row), d1 = load_chunk(c.a32, 7, row);
		dens[0] = d0.x; dens[1] = d0.y; dens[2] = d0.z; dens[3] = d0.w; dens[4] = d1.x; dens[5] = d1.y; dens[6] = d1.z; dens[7] = d1.w;
	}
	tile_sync(c);  // every warp's first layer has read its operand
	if (density_only) return;
	if (release && row == 0) mbar_arrive(release);
	// rgb-network input: columns 0-15 = density MLP output, 16-31 = SH (nerf_network_full.h:52,67,79)
	__half2 sh[8];
	encode_sh4(dw, sh);  // tcnn SphericalHarmonics of the (mapped) direction
	store_chunk(c.a32, 0, row, make_uint4(dens[0], dens[1], dens[2], dens[3]));
	store_chunk(c.a32, 1, row, make_uint4(dens[4], dens[5], dens[6], dens[7]));
	store_chunk(c.a32, 2, row, make_uint4(pack_h2(sh[0]), pack_h2(sh[1]), pack_h2(sh[2]), pack_h2(sh[3])));
	store_chunk(c.a32, 3, row, make_uint4(pack_h2(sh[4]), pack_h2(sh[5]), pack_h2(sh[6]), pack_h2(sh[7])));
	fence_async_smem();
	tile_sync(c);
#pragma unroll 1
	for (uint32_t h = 0; h < 2; ++h) {
		Acc<64, ACC16> x, y;
		Acc<16, ACC16> o;
		layer_ss<64, 32, ACC16>(x.r, a32 + h * 64 * 16, w + W3_OFF);  // L3: 32 -> 64
		layer_rs<64, 64, ACC16>(y.r, x.r, w + W4_OFF);                // L4: 64 -> 64
		layer_rs<16, 64, ACC16>(o.r, y.r, w + W5_OFF);                // L5: 64 -> 16
		store_out16<ACC16>(c.a32, 4, row, h, o.r);
	}
	__syncwarp();
	{
		const uint4 r0 = load_chunk(c.a32, 4, row), r1 = load_chunk(c.a32, 5, row);
		rgb[0] = r0.x; rgb[1] = r0.y; rgb[2] = r0.z; rgb[3] = r0.w; rgb[4] = r1.x; rgb[5] = r1.y; rgb[6] = r1.z; rgb[7] = r1.w;
	}
	tile_sync(c);
}

}  // namespace tc
}  // namespace nsb
