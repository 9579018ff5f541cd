// nsb_kernels.cu — kernels of the H100-native NeRFshop render path and the C ABI on top of them.
//
// The product kernel is k_render_fused: ONE persistent launch per frame that replaces the reference's
// per-round pipeline (compact -> generate inputs -> [residuals] -> inference -> [map_rays] -> inference ->
// composite, >= 12 launches + 3 host syncs per round, testbed_nerf.cu:2812-2990) and its 4.6 GB of
// scratch: ray state lives in registers and shared memory, samples go march -> deform -> hash encode -> wgmma MLP ->
// composite without touching HBM, and finished rays are shaded straight into the framebuffer.
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <ctime>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "../../include/nerfshop_b200.h"
#include "nsb_device.cuh"
#include "nsb_tc.cuh"

using namespace nsb;

// =====================================================================================================
// fused persistent renderer
// =====================================================================================================
struct RayRec { uint32_t pix; float t; };  // a ray that entered the AABB and found occupied space: pixel + first sample t

enum { ST_RAYS = 0, ST_ALIVE = 1, ST_HIT = 2, ST_SAMPLES = 3, ST_OLD = 4, ST_ROUNDS = 5, ST_CYC_ACQUIRE = 6, ST_CYC_ENCODE = 7, ST_CYC_MLP = 8,
       ST_CYC_COMPOSITE = 9, ST_CYC_TOTAL = 10, ST_TILES = 11, ST_N = 12 };
constexpr int DDA_BUDGET = 8;   // empty voxels a lane may skip per MLP round before it yields (latency bound of a round)
constexpr int REFILL_THR = 2;   // the free lanes of a warp refill once at most this many of its rays are alive

// tile slot -> pixel: the four warps of a 16x8 tile each cover an 8x4 block so that the 32 lanes of a warp stay
// spatially compact (coherent hash-grid and occupancy lookups)
__device__ __forceinline__ bool tile_pixel(const DevFrame& f, uint32_t tile, uint32_t slot, uint32_t& px, uint32_t& py) {
	uint32_t tx = tile % (uint32_t)f.tiles_x, ty = tile / (uint32_t)f.tiles_x;
	uint32_t b = slot >> 5, l = slot & 31u;
	px = tx * TILE_W + (b & 1u) * 8u + (l & 7u);
	py = ty * TILE_H + (b >> 1) * 4u + (l >> 3);
	return px < (uint32_t)f.W && py < (uint32_t)f.H;
}

// Stage 1 (massively parallel, one thread per pixel of this rank's tiles):
// init_rays_with_payload_kernel_nerf (testbed_nerf.cu:2512) + advance_pos_nerf (:557) + the alive-ray compaction
// of compact_kernel_nerf (:2485), with warp-aggregated atomics instead of one global atomic per ray.
// The long empty-space walk to a ray's first occupied sample is a serial chain of dependent occupancy loads;
// here it is hidden by running every ray of the frame concurrently instead of stalling an MLP round.
// GENERAL: frames with lens distortion / a distortion map / depth of field (f.general_camera), an environment map or the Distortion render mode.
// Their rays cost a Newton iteration or a sincosf to generate, so the queued ones are handed to the persistent renderer in `ray_od` (origin and
// direction, 6 floats per queue slot) instead of being re-derived from the pixel index there; the common pinhole path stays as lean as it was.
template <bool GENERAL>
__global__ void __launch_bounds__(256) k_prepare_rays(const DevFrame f, const uint8_t* __restrict__ bitfield, float4* __restrict__ fb, float* __restrict__ depth_out,
                                                      RayRec* __restrict__ list, float* __restrict__ ray_od, uint32_t* __restrict__ n_queued, uint32_t n_local_pixels,
                                                      unsigned long long* __restrict__ stats) {
	__shared__ uint32_t spread7[128];
	fill_spread7(spread7);
	__syncthreads();
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	bool queued = false, is_ray = false, entered = false;
	uint32_t pix = 0;
	float t = 0.0f;
	Ray r;
	if (i < n_local_pixels) {
		uint32_t tile = (uint32_t)f.tile_rank + (i / (uint32_t)TILE_PIXELS) * (uint32_t)f.tile_world;
		uint32_t px, py;
		if (tile_pixel(f, tile, i % (uint32_t)TILE_PIXELS, px, py)) {
			is_ray = true;
			pix = px + (uint32_t)f.W * py;
			depth_out[pix] = 1e10f;  // :2581
			bool inside;
			if constexpr (GENERAL) {
				inside = f.general_camera ? make_ray_general(f, px, py, r) : make_ray(f, px, py, r);
				if (f.envmap) fb[pix] = read_envmap(f.envmap, f.env_w, f.env_h, r.d);  // every pixel, before the AABB test (:2581-2583)
				if (inside && f.mode == NSB_RENDER_DISTORTION) {  // :2596-2607: the map itself, written by ray initialisation; the ray is not traced
					float dx = 0.5f, dy = 0.5f;
					if (f.distortion) {
						read_image2(f.distortion, f.dist_w, f.dist_h, ((float)px + 0.5f) / (float)f.W, ((float)py + 0.5f) / (float)f.H, dx, dy);
						dx = dx * 50.0f + 0.5f; dy = dy * 50.0f + 0.5f;
					}
					fb[pix] = make_float4(dx, dy, 0.5f, 1.0f);
					depth_out[pix] = 1.0f;
					inside = false;
				}
			} else {
				inside = make_ray(f, px, py, r);
			}
			if (inside) {
				entered = true;
				V3 idir = v3(__frcp_rn(r.d.x), __frcp_rn(r.d.y), __frcp_rn(r.d.z));
				t = fma_(ld_random_val(f.spp, pix * 786433u), calc_dt(r.t, f.cone), r.t);  // advance_pos_nerf :585
				float dt; V3 pos; uint32_t mip, cell;
				queued = next_occupied(f, bitfield, spread7, r.o, r.d, idir, t, dt, pos, mip, cell);
			}
		}
	}
	const unsigned lane = threadIdx.x & 31u;
	unsigned m = __ballot_sync(0xffffffffu, queued);
	unsigned mr = __ballot_sync(0xffffffffu, is_ray), me = __ballot_sync(0xffffffffu, entered);
	uint32_t base = 0;
	if (lane == 0) {
		if (m) base = atomicAdd(n_queued, (uint32_t)__popc(m));
		if (mr) atomicAdd(stats + ST_RAYS, (unsigned long long)__popc(mr));
		if (me) atomicAdd(stats + ST_ALIVE, (unsigned long long)__popc(me));
	}
	base = __shfl_sync(0xffffffffu, base, 0);
	if (queued) {
		RayRec rr;
		rr.pix = pix;
		rr.t = t;
		const uint32_t slot = base + __popc(m & ((1u << lane) - 1u));
		list[slot] = rr;
		if constexpr (GENERAL) {
			if (ray_od) {
				float* od = ray_od + 6 * (size_t)slot;
				od[0] = r.o.x; od[1] = r.o.y; od[2] = r.o.z; od[3] = r.d.x; od[4] = r.d.y; od[5] = r.d.z;
			}
		}
	}
}

// grid features of one sample -> this thread's row of the A operand (4 chunks x 8 fp16)
// Code size matters here: the fused kernel's hot loop has to live in the SM's instruction cache (a fully unrolled version
// stalls on instruction fetch). One loop body = 2 levels (16 gathers in flight per thread), 8 iterations.
#ifndef NSB_ENC_NL
#define NSB_ENC_NL 2  // levels per loop iteration (8*NL gathers in flight per thread)
#endif
// IN_RANGE: grid_index's shortcut (nsb_device.cuh); only k_render_fused passes true, for frames where render_in_range holds.
template <bool IN_RANGE = false>
__device__ __forceinline__ void encode_to_a32(uint8_t* a32, const DevModel& m, bool valid, V3 pw, uint32_t row) {
	constexpr int NL = NSB_ENC_NL;
#pragma unroll 1
	for (int g = 0; g < MAX_LEVELS / NL; ++g) {
		__half2 h[NL];
#pragma unroll
		for (int j = 0; j < NL; ++j) h[j] = __floats2half2_rn(0.0f, 0.0f);
		if (valid) {
			uint32_t mode = m.pair_mode[(NL * g) / 2];  // uniform
			if (NL == 4 && m.pair_mode[(NL * g) / 2 + 1] != mode) mode = 2;
			if (mode == 1) encode_levels<NL, 1, IN_RANGE>(m.levels + NL * g, m.grid, pw.x, pw.y, pw.z, h);
			else if (mode == 0) encode_levels<NL, 0, IN_RANGE>(m.levels + NL * g, m.grid, pw.x, pw.y, pw.z, h);
			else encode_levels<NL, 2, IN_RANGE>(m.levels + NL * g, m.grid, pw.x, pw.y, pw.z, h);
		}
		// levels NL*g .. NL*g+NL-1 = fp16 features 2*NL*g ..: NL*4 bytes of this row's k-chunk (NL*g)/4
		uint8_t* dst = a32 + ((NL * g) >> 2) * (tc::ROWS * 16) + tc::phys_row(row) * 16 + ((NL * g) & 3) * 4;
		if (NL == 2) *reinterpret_cast<uint2*>(dst) = make_uint2(tc::pack_h2(h[0]), tc::pack_h2(h[1]));
		else *reinterpret_cast<uint4*>(dst) = make_uint4(tc::pack_h2(h[0]), tc::pack_h2(h[1]), tc::pack_h2(h[NL > 2 ? 2 : 0]), tc::pack_h2(h[NL > 3 ? 3 : 0]));
	}
}

// The loop of the one-tile network kernels (one CTA = 128 threads = one tile of 128 rows, tc::TileSmem of dynamic shared memory,
// grid-stride over the n_padded rows). sample(i, pw, dw) runs for valid rows (i < n) only and sets the row's warped position and
// direction; the other rows keep the origin and dw_default. emit(i, valid, pw, dens, rgbo) runs for every row i < n_padded, the
// padding included, with the network's outputs (density_only: the density MLP alone). n_padded must be a multiple of 128: emit is
// called for every row of every tile, so a partial last tile would reach past n_padded.
// The loop walks tile indices, not row bases: a row base stepped by gridDim.x * 128 wraps past 2^32 when n_padded is within one stride
// of it, and the CTA would start over. A tile index stays below 2^25 and its step below 2^16, so it cannot wrap.
template <bool ACC16, typename Sample, typename Emit>
__device__ __forceinline__ void network_tiles(const DevModel& m, uint32_t n, uint32_t n_padded, bool density_only, V3 dw_default, Sample sample, Emit emit) {
	extern __shared__ __align__(128) uint8_t smem_raw[];
	tc::TileSmem& S = *reinterpret_cast<tc::TileSmem*>(smem_raw);
	const uint32_t tid = threadIdx.x;
	tc::tile_setup(S, m.w_image);
	const uint32_t n_tiles = n_padded / 128u;
	for (uint32_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
		const uint32_t i = t * 128u + tid;
		const bool valid = i < n;
		V3 pw = v3(0, 0, 0), dw = dw_default;
		if (valid) sample(i, pw, dw);
		uint32_t dens[8], rgbo[8];
		encode_to_a32(S.a32, m, valid, pw, tid);
		tc::run_network<ACC16>(tc::single_tile_ctx(S), dw, density_only, dens, rgbo);
		emit(i, valid, pw, dens, rgbo);
	}
}

__device__ __forceinline__ float h_lo(uint32_t packed) { return __half2float(__ushort_as_half((unsigned short)(packed & 0xffffu))); }
__device__ __forceinline__ float h_hi(uint32_t packed) { return __half2float(__ushort_as_half((unsigned short)(packed >> 16))); }

// Stage 2 (persistent; a tile = 128 threads = 128 ray slots = 128 MMA rows, RENDER_TILES tiles per CTA): every round each live ray contributes
// ONE sample; samples go deform -> hash encode -> wgmma MLPs -> composite inside the SM; a finished ray is shaded
// into the framebuffer and its slot refilled from the queue (warp-convergent fetch of consecutive entries, so rays that
// were refilled together — neighbouring pixels that die on the same surface — stay together in a warp).
// Per-slot ray state parked in shared memory (SoA: lane-contiguous, conflict-free). Only the acquire and composite phases
// touch it, so it does not occupy registers while the thread gathers hash-grid features and walks the MLP layers.
enum { R_OX = 0, R_OY, R_OZ, R_DX, R_DY, R_DZ, R_T, R_CR, R_CG, R_CB, R_CA, R_DEPTH, R_MAXW, R_FIELDS };
// One CTA per SM holds render_tiles(OPS, ACC16) independent tiles (a tile = 128 threads = 128 ray slots = one warpgroup). The tiles share
// the 20 KB weight image — four separate CTAs would hold four copies — which matters because shared memory is carved out of the same
// 256 KB as the L1 that serves the hash-grid gathers.
// How many: the register file's worth, per instantiation. Frames without operators and fp16 accumulators (the default): 7 tiles (28 warps
// per SM, 72 registers per thread, 122 KB of shared memory), no spills. fp32 accumulators: 6 tiles (80 registers, 20 B of spill stores
// per thread; capped at 72 they spill 66-106 B and ptxas serialises the wgmma chain). Frames with operators carry the deform / membrane
// state: 5 tiles (96 registers; 86-98 B of spill stores per thread; six tiles at 80 registers spill twice that and measured slower).
constexpr int RENDER_TILES_ACC16 = 7, RENDER_TILES = 6, RENDER_TILES_OPS = 5;
struct TileBlock {
	uint8_t a32[tc::A32_BYTES];  // run_network's operand space
	float ray[R_FIELDS][128];
};
template <int TILES>
struct __align__(128) RenderSmemT {
	uint8_t w[tc::W_BYTES];
	TileBlock tile[TILES];
	uint32_t spread7[128];  // fill_spread7: the march's Morton table
	uint64_t w_bar;
	uint32_t pad[2];
};
__host__ __device__ constexpr int render_tiles(bool ops, bool acc16) { return ops ? RENDER_TILES_OPS : acc16 ? RENDER_TILES_ACC16 : RENDER_TILES; }
static_assert(RENDER_TILES_ACC16 >= 1 && RENDER_TILES_ACC16 <= 8 && RENDER_TILES >= 1 && RENDER_TILES <= 8 && RENDER_TILES_OPS >= 1 && RENDER_TILES_OPS <= 8,
              "1..8 tiles (warpgroups) per CTA");

// OPS = false: the instantiation for frames without edit operators (f.apply_ops == 0 or no operator uploaded) carries none of the deform /
// membrane code in its hot loop (the loop has to fit the instruction cache).
// ACC16: the MLP accumulator policy (nsb_set_mlp_accumulator): fp16 wgmma accumulators, like the reference's wmma __half fragments.
// IN_RANGE (only with OPS = false): the hash grid takes grid_index's one-subtraction modulo; the host picks it where render_in_range holds.
template <bool OPS, bool ACC16, bool IN_RANGE>
__global__ void __launch_bounds__(128 * render_tiles(OPS, ACC16), 1) k_render_fused(const DevFrame f, const DevModel m, const uint8_t* __restrict__ bitfield,
                                                      const DevOp* __restrict__ ops, const int n_ops, const int any_poisson,
                                                      float4* __restrict__ fb, float* __restrict__ depth_out, const RayRec* __restrict__ list,
                                                      const float* __restrict__ ray_od, const uint32_t* __restrict__ n_queued_ptr, uint32_t* fetch_counter,
                                                      unsigned long long* __restrict__ stats) {
	extern __shared__ __align__(128) uint8_t smem_raw[];
	constexpr int TILES = render_tiles(OPS, ACC16);
	using RenderSmem = RenderSmemT<TILES>;
	RenderSmem& RS = *reinterpret_cast<RenderSmem*>(smem_raw);
	const uint32_t tid = threadIdx.x & 127u;      // slot / row within the tile
	const uint32_t tile = threadIdx.x >> 7;
	TileBlock& TB = RS.tile[tile];
	const uint32_t lane = tid & 31u;
	if (blockIdx.x * 128u * TILES >= *n_queued_ptr && blockIdx.x > 0) return;  // nothing this CTA could ever fetch

	// CTA setup: one bulk-TMA copy of the weight image
	tc::load_weights(RS.w, &RS.w_bar, m.w_image);
	fill_spread7(RS.spread7);
	__syncthreads();
	tc::mbar_wait(&RS.w_bar, 0);
	tc::TileCtx C;
	C.a32 = TB.a32; C.w_addr = tc::smem_u32(RS.w); C.row = tid;
	C.bar_id = 1 + tile;

	constexpr bool ops_on = OPS;  // the host picks the instantiation: f.apply_ops && n_ops > 0
	static_assert(!(OPS && IN_RANGE), "operators map samples anywhere: their frames take the exact grid index");

	// what stays in registers across a round
	bool alive = false, exhausted = false;  // exhausted is warp-uniform: the queue had nothing left when this warp last asked
	uint32_t pix = 0, n_steps = 0;
	uint32_t c_hit = 0, c_samples = 0, c_old = 0;
	// phase profile (thread 0 of each tile; a handful of clock reads per round): diagnostic builds only (-DNSB_PROFILE), the
	// product build keeps the registers and issue slots (nsb_debug_counters then reports rounds and tiles only)
#ifdef NSB_PROFILE
#define NSB_CLOCK() clock64()
	long long cyc_acq = 0, cyc_enc = 0, cyc_mlp = 0, cyc_comp = 0;
	const long long cyc_start = clock64();
#else
#define NSB_CLOCK() 0ll
#endif
	uint32_t n_rounds = 0;

	// shade_kernel_nerf (:2464-2482) for the ray this thread just finished (compact_kernel_nerf :2503 filter)
	auto finish = [&](bool left_aabb, float cr, float cg, float cb, float ca, float ray_depth) {
		alive = false;
		if (!(ca > 0.001f)) return;
		++c_hit;
		float r = cr, g = cg, b = cb, a = ca;
		if (f.mode == NSB_RENDER_COST) {
			float col = (float)(n_steps + (left_aabb ? 1u : 0u)) / 128.0f;
			r = g = b = col;
			a = 1.0f;
		}
		if (!f.linear_colors && f.mode == NSB_RENDER_SHADE) { r = srgb_to_linear(r); g = srgb_to_linear(g); b = srgb_to_linear(b); }
		float4 prev = fb[pix];
		float om = 1.0f - a;
		fb[pix] = make_float4(__fmaf_rn(prev.x, om, r), __fmaf_rn(prev.y, om, g), __fmaf_rn(prev.z, om, b), __fmaf_rn(prev.w, om, a));
		if (a > 0.2f) depth_out[pix] = ray_depth;
	};

	for (;;) {
		if (!tc::tile_any(C, alive || !exhausted)) break;
#ifdef NSB_PROFILE
		const long long c0 = clock64();
#endif

		// ---- acquire one occupied sample for this thread (refill the ray slot when it is free) ----
		bool has_sample = false;
		float dt = 0.0f;
		V3 pos = v3(0, 0, 0), dw = v3(0.5f, 0.5f, 0.5f);
		{
			int budget = DDA_BUDGET;
			V3 ro = v3(TB.ray[R_OX][tid], TB.ray[R_OY][tid], TB.ray[R_OZ][tid]);
			V3 rd = v3(TB.ray[R_DX][tid], TB.ray[R_DY][tid], TB.ray[R_DZ][tid]);
			float t = TB.ray[R_T][tid];
			// Refill (warp-convergent). Free lanes wait until the warp is down to <= REFILL_THR live rays, then take consecutive queue
			// entries (neighbouring pixels) in one claim, so the lanes of a warp gather from the same few hash-grid cells on the coarse
			// and middle levels instead of 32 unrelated cache lines per instruction.
			{
				const unsigned alive_m = __ballot_sync(0xffffffffu, alive);
				const unsigned want = exhausted ? 0u : ~alive_m;
				if (want && __popc(alive_m) <= REFILL_THR) {
					// read at each refill (an L1 hit), not held across the round: at 72 registers a held copy is spilled
					const uint32_t n_queued = __ldca(n_queued_ptr);
					const uint32_t need = (uint32_t)__popc(want), rank = (uint32_t)__popc(want & ((1u << lane) - 1u));
					uint32_t base = 0;
					if (lane == 0) base = atomicAdd(fetch_counter, need);
					base = __shfl_sync(0xffffffffu, base, 0);
					exhausted = base + need > n_queued;  // a short claim: the queue has nothing left for this warp
					const uint32_t qi = base + rank;     // free lane of free-rank `rank`
					if (!alive && qi < n_queued) {
						const RayRec rr = list[qi];
						pix = rr.pix;
						if (ray_od) {  // a general-camera frame: k_prepare_rays<true> left the ray next to its queue entry
							const float* od = ray_od + 6 * (size_t)qi;
							ro = v3(od[0], od[1], od[2]); rd = v3(od[3], od[4], od[5]);
						} else {
							Ray r;
							make_ray(f, pix % (uint32_t)f.W, pix / (uint32_t)f.W, r);
							ro = r.o; rd = r.d;
						}
						t = rr.t;
						TB.ray[R_OX][tid] = ro.x; TB.ray[R_OY][tid] = ro.y; TB.ray[R_OZ][tid] = ro.z;
						TB.ray[R_DX][tid] = rd.x; TB.ray[R_DY][tid] = rd.y; TB.ray[R_DZ][tid] = rd.z;
						TB.ray[R_CR][tid] = 0.0f; TB.ray[R_CG][tid] = 0.0f; TB.ray[R_CB][tid] = 0.0f; TB.ray[R_CA][tid] = 0.0f;
						TB.ray[R_DEPTH][tid] = 0.0f; TB.ray[R_MAXW][tid] = 0.0f;
						n_steps = 0;
						alive = true;
					}
				}
			}
			for (;;) {
				if (!alive) break;
				if (n_steps >= MARCH_ITER - 1) { alive = false; continue; }  // still marching after MARCH_ITER steps: dropped (:2812)
				// __frcp_rn(x) == __fdiv_rn(1, x) bit for bit (the correctly rounded 1/x, ±0 -> ±inf), two instructions shorter
				const V3 idir = v3(__frcp_rn(rd.x), __frcp_rn(rd.y), __frcp_rn(rd.z));
				const MarchResult mr = next_occupied_budget(f, bitfield, RS.spread7, ro, rd, idir, t, dt, pos, budget);
				if (mr == MARCH_FOUND) { has_sample = true; break; }
				if (mr == MARCH_EXIT) {
					finish(true, TB.ray[R_CR][tid], TB.ray[R_CG][tid], TB.ray[R_CB][tid], TB.ray[R_CA][tid], TB.ray[R_DEPTH][tid]);
					continue;
				}
				break;  // MARCH_PENDING: resume next round
			}
			if (has_sample) {
				dw = warp_direction(rd);
				t = add(t, dt);
			}
			if (alive) TB.ray[R_T][tid] = t;
		}

		// ---- network inputs: generate_next_nerf_network_inputs :690 ----
		V3 pw = v3(0, 0, 0);
		float dtw = 0.0f;
		bool empty = false;
		Membrane mem;
		mem.op = -1; mem.tet = -1; mem.dob = 0.0f; mem.drb = 0.0f;
		bool need_old = false;
		V3 pw_old = pw;
		if (has_sample) {
			pw = (!OPS && f.tinv_exact) ? warp_position_pow2(pos, f.tmin, f.tinv) : warp_position(pos, f.tmin, f.tmax);  // uniform branch; with operators it raised the spills
			dtw = warp_dt(dt);
			++n_steps;
			++c_samples;
			if (ops_on) {
				if (any_poisson) {  // membrane residuals are evaluated in deformed space (:2867-2883)
					poisson_one(ops, n_ops, pw, mem);
					need_old = mem.dob > 1e-9f && f.poisson_target;
				}
				pw_old = pw;
				map_one(ops, n_ops, pw, dw, empty);  // backward map into canonical space (:2896-2904)
			}
		}

		// ---- encode + fused MLPs. Pass 0 (rare) is the "old" density on the un-mapped position: the reference runs a second
		// full inference every round (:2892) but only the membrane's poisson-target blend ever reads it (:773), so it is
		// evaluated only in rounds where some lane needs it, density MLP only. Pass 1 is the real sample. One code copy.
		float sigma_old_raw = 0.0f;
		uint32_t dens[8], rgbo[8];
		int first_pass = 1;
		if (ops_on && any_poisson && f.poisson_target) first_pass = tc::tile_any(C, need_old) ? 0 : 1;
#ifdef NSB_PROFILE
		const long long c1 = clock64();
		long long enc_cycles = 0;
#endif
#pragma unroll 1
		for (int pass = first_pass; pass < 2; ++pass) {
			const bool old_pass = pass == 0;
#ifdef NSB_PROFILE
			const long long e0 = clock64();
#endif
			encode_to_a32<IN_RANGE>(TB.a32, m, old_pass ? need_old : has_sample, old_pass ? pw_old : pw, tid);
#ifdef NSB_PROFILE
			enc_cycles += clock64() - e0;
#endif
			tc::run_network<ACC16>(C, dw, old_pass, dens, rgbo);
			if (old_pass) {
				sigma_old_raw = h_lo(dens[0]);
				if (need_old) ++c_old;
			}
		}
#ifdef NSB_PROFILE
		const long long c2 = c1 + enc_cycles;
		const long long c3 = clock64();
#endif

		// ---- composite_kernel_nerf :750-955, split in two: what depends on the sample alone, then the ray's running sums ----
		float s_alpha = 0.0f, s_e[3] = {0.0f, 0.0f, 0.0f}, s_z = 0.0f;
		float s_mask = 1.0f;  // glow_mode's mask_to_alpha: multiplies the sample's weight (:877-879)
		if (has_sample) {
			const V3 cam_fwd = v3(f.cam1[6], f.cam1[7], f.cam1[8]);
			V3 cpos = unwarp_position(pw, f.tmin, f.tmax);
			float dtu = unwarp_dt(dtw);
			float sigma = network_to_density(h_lo(dens[0]), f.density_act);  // row 3 = density MLP out[0] (extract_density)
			float alpha;
			const bool membrane = OPS && mem.dob > 1e-9f;
			if (empty) {
				alpha = 0.0f;
			} else if (membrane) {
				float val;
				if (f.poisson_target) {
					float target = network_to_density(sigma_old_raw, f.density_act);
					val = fminf(fmaxf(target, sigma), sigma + mem.drb);
				} else {
					val = sigma + mem.drb;
				}
				alpha = 1.0f - __expf(-val * dtu);
			} else {
				alpha = 1.0f - __expf(-sigma * dtu);
			}
			if (f.show_accel) alpha = 1.0f;  // show_accel >= 0: the occupancy cells themselves are drawn (:788-790)
			float rgb[3] = {network_to_rgb(h_lo(rgbo[0]), f.rgb_act), network_to_rgb(h_hi(rgbo[0]), f.rgb_act), network_to_rgb(h_lo(rgbo[1]), f.rgb_act)};
			if (f.glow_mode) {  // :807-903, before the mode overrides
				const float4 gl = glow_apply(f.glow_mode, f.glow_y_cutoff, cpos, v3(f.cam1[9], f.cam1[10], f.cam1[11]), rgb[0], rgb[1], rgb[2]);
				rgb[0] = gl.x; rgb[1] = gl.y; rgb[2] = gl.z; s_mask = gl.w;
			}
			if (f.mode != NSB_RENDER_SHADE) {
				const V3 ro = v3(TB.ray[R_OX][tid], TB.ray[R_OY][tid], TB.ray[R_OZ][tid]);
				if (f.mode == NSB_RENDER_AO) { rgb[0] = rgb[1] = rgb[2] = alpha; }
				else if (f.mode == NSB_RENDER_POSITIONS && f.show_accel) {  // one random colour per occupancy cell (:913-923)
					const uint32_t mip = (uint32_t)max(f.min_mip, mip_from_pos(cpos));
					const float res = (float)(GRIDSIZE >> mip);
					const int ix = (int)mul(cpos.x, res), iy = (int)mul(cpos.y, res), iz = (int)mul(cpos.z, res);
					Pcg32 rng;  // tcnn::default_rng_t rng(seed): pcg32::seed(initstate, initseq = 1)
					rng.state = 0; rng.inc = 3;
					rng.next_uint();
					rng.state += (uint64_t)(int64_t)(ix + iy * 232323 + iz * 727272);
					rng.next_uint();
					rgb[0] = fma_(-(float)mip, 0.25f, 1.0f);
					rgb[1] = rng.next_float();
					rgb[2] = rng.next_float();
				}
				else if (f.mode == NSB_RENDER_POSITIONS) { rgb[0] = (cpos.x - 0.5f) / 2.0f + 0.5f; rgb[1] = (cpos.y - 0.5f) / 2.0f + 0.5f; rgb[2] = (cpos.z - 0.5f) / 2.0f + 0.5f; }
				else if (f.mode == NSB_RENDER_DEPTH) { float z = dot3(cam_fwd, vsub(cpos, ro)) * f.depth_scale; rgb[0] = rgb[1] = rgb[2] = z; }
				else if (f.mode == NSB_RENDER_DISTANCE) { V3 q = vsub(cpos, ro); float z = sqrtf(dot3(q, q)) * f.depth_scale; rgb[0] = rgb[1] = rgb[2] = z; }
				else if (f.mode == NSB_RENDER_STEPSIZE) { float wdt = warp_dt(dtu); rgb[0] = rgb[1] = rgb[2] = wdt; }
			}
			if (membrane) {
				float alpha_N = 1.0f - __expf(-sigma * dtu);
				float alpha_R = 1.0f - __expf(-mem.dob * dtu);
				float w_N = alpha_N / (alpha_N + alpha_R), w_R = alpha_R / (alpha_N + alpha_R);
				float res[3];
				membrane_rgb(ops, mem, unwarp_direction(dw), res);
				rgb[0] = __fmaf_rn(w_R, res[0], w_N * rgb[0]);
				rgb[1] = __fmaf_rn(w_R, res[1], w_N * rgb[1]);
				rgb[2] = __fmaf_rn(w_R, res[2], w_N * rgb[2]);
			}
			s_alpha = alpha; s_e[0] = rgb[0]; s_e[1] = rgb[1]; s_e[2] = rgb[2];
			s_z = dot3(cam_fwd, vsub(cpos, v3(f.cam1[9], f.cam1[10], f.cam1[11])));
		}
		if (has_sample) {
			const float sat = 1.0f - f.min_T;  // rendering_min_transmittance test of composite_kernel_nerf :951
			float cr = TB.ray[R_CR][tid], cg = TB.ray[R_CG][tid], cb = TB.ray[R_CB][tid], ca = TB.ray[R_CA][tid];
			float ray_depth = TB.ray[R_DEPTH][tid], max_weight = TB.ray[R_MAXW][tid];
			auto accumulate = [&](const float alpha, const float e0, const float e1, const float e2, const float z) {
				float T = 1.0f - ca;
				float weight = alpha * T;
				cr = __fmaf_rn(e0, weight, cr);
				cg = __fmaf_rn(e1, weight, cg);
				cb = __fmaf_rn(e2, weight, cb);
				ca += weight;
				if (weight > max_weight) {
					max_weight = weight;
					ray_depth = z;
				}
				if (ca > sat) {
					float a = ca;
					cr = __fdiv_rn(cr, a); cg = __fdiv_rn(cg, a); cb = __fdiv_rn(cb, a); ca = __fdiv_rn(ca, a);
					finish(false, cr, cg, cb, ca, ray_depth);
				}
			};
			if (f.glow_mode & 4) {
				// mask_to_alpha: weight *= mask (a separate copy so that the unmasked expression — and its FMA contraction — stays exactly the reference's)
				float T = 1.0f - ca;
				float weight = s_alpha * T;
				weight *= s_mask;
				cr = __fmaf_rn(s_e[0], weight, cr);
				cg = __fmaf_rn(s_e[1], weight, cg);
				cb = __fmaf_rn(s_e[2], weight, cb);
				ca += weight;
				if (weight > max_weight) { max_weight = weight; ray_depth = s_z; }
				if (ca > sat) {
					float a = ca;
					cr = __fdiv_rn(cr, a); cg = __fdiv_rn(cg, a); cb = __fdiv_rn(cb, a); ca = __fdiv_rn(ca, a);
					finish(false, cr, cg, cb, ca, ray_depth);
				}
			} else {
				accumulate(s_alpha, s_e[0], s_e[1], s_e[2], s_z);
			}
			if (alive) {
				TB.ray[R_CR][tid] = cr; TB.ray[R_CG][tid] = cg; TB.ray[R_CB][tid] = cb; TB.ray[R_CA][tid] = ca;
				TB.ray[R_DEPTH][tid] = ray_depth; TB.ray[R_MAXW][tid] = max_weight;
			}
		}
#ifdef NSB_PROFILE
		cyc_acq += c1 - c0; cyc_enc += c2 - c1; cyc_mlp += c3 - c2; cyc_comp += clock64() - c3;
#endif
		++n_rounds;
	}

	if (tid == 0) {
		atomicAdd(stats + ST_ROUNDS, (unsigned long long)n_rounds);
#ifdef NSB_PROFILE
		atomicAdd(stats + ST_CYC_ACQUIRE, (unsigned long long)cyc_acq);
		atomicAdd(stats + ST_CYC_ENCODE, (unsigned long long)cyc_enc);
		atomicAdd(stats + ST_CYC_MLP, (unsigned long long)cyc_mlp);
		atomicAdd(stats + ST_CYC_COMPOSITE, (unsigned long long)cyc_comp);
		atomicAdd(stats + ST_CYC_TOTAL, (unsigned long long)(clock64() - cyc_start));
#endif
		atomicAdd(stats + ST_TILES, 1ull);
	}

	// counters: warp reduce, one atomic per warp
	unsigned long long c[3] = {c_hit, c_samples, c_old};  // per-thread counts fit 32 bits (one thread composites < 2^32 samples per frame)
	const int slot[3] = {ST_HIT, ST_SAMPLES, ST_OLD};
#pragma unroll
	for (int k = 0; k < 3; ++k) {
		unsigned long long v = c[k];
		for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
		if (lane == 0 && v) atomicAdd(stats + slot[k], v);
	}
}

// =====================================================================================================
// operator-level kernels (same device code as the fused renderer)
// =====================================================================================================
// NerfNetwork::inference_mixed_precision / ::density on a flat batch: one CTA = 128 samples.
template <bool DENSITY_ONLY, bool ACC16>
__global__ void __launch_bounds__(128) k_inference(const DevModel m, const float* __restrict__ coords, uint32_t n, __half* __restrict__ out,
                                                   uint32_t n_padded) {
	network_tiles<ACC16>(m, n, n_padded, DENSITY_ONLY, v3(0.5f, 0.5f, 0.5f), [&](uint32_t i, V3& pw, V3& dw) {
		pw = v3(coords[7 * (size_t)i], coords[7 * (size_t)i + 1], coords[7 * (size_t)i + 2]);
		dw = v3(coords[7 * (size_t)i + 4], coords[7 * (size_t)i + 5], coords[7 * (size_t)i + 6]);
	}, [&](uint32_t i, bool, V3, const uint32_t* dens, const uint32_t* rgbo) {  // every row: the padding gets the output of the zero input
		const uint32_t* src = DENSITY_ONLY ? dens : rgbo;
#pragma unroll
		for (int k = 0; k < 8; ++k) {
			out[(size_t)(2 * k) * n_padded + i] = __ushort_as_half((unsigned short)(src[k] & 0xffffu));
			out[(size_t)(2 * k + 1) * n_padded + i] = __ushort_as_half((unsigned short)(src[k] >> 16));
		}
		if (!DENSITY_ONLY) out[(size_t)3 * n_padded + i] = __ushort_as_half((unsigned short)(dens[0] & 0xffffu));  // extract_density
	});
}

// tcnn GridEncoding inference alone: fp16 [32 x n_padded] row-major, same loop body as the fused kernel.
__global__ void __launch_bounds__(256) k_encode(const DevModel m, const float* __restrict__ coords, uint32_t n, __half* __restrict__ out, uint32_t n_padded) {
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	float x = coords[7 * (size_t)i], y = coords[7 * (size_t)i + 1], z = coords[7 * (size_t)i + 2];
#pragma unroll 1
	for (uint32_t g = 0; g < MAX_LEVELS / 2; ++g) {
		__half2 v[2];
		const uint32_t mode = m.pair_mode[g];  // uniform
		if (mode == 1) encode_levels<2, 1>(m.levels + 2 * g, m.grid, x, y, z, v);
		else if (mode == 0) encode_levels<2, 0>(m.levels + 2 * g, m.grid, x, y, z, v);
		else encode_levels<2, 2>(m.levels + 2 * g, m.grid, x, y, z, v);
#pragma unroll
		for (uint32_t j = 0; j < 2; ++j) {
			out[(size_t)(4 * g + 2 * j) * n_padded + i] = __low2half(v[j]);
			out[(size_t)(4 * g + 2 * j + 1) * n_padded + i] = __high2half(v[j]);
		}
	}
}

// EditOperator::map_rays for operators [0, n_ops) of `ops` in reverse order; the mask is only ever SET (the caller clears it, testbed_nerf.cu:2898)
__global__ void k_map_rays(const DevOp* __restrict__ ops, int n_ops, float* __restrict__ coords, uint8_t* __restrict__ empty_mask, uint32_t n) {
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	V3 pw = v3(coords[7 * (size_t)i], coords[7 * (size_t)i + 1], coords[7 * (size_t)i + 2]);
	V3 dw = v3(coords[7 * (size_t)i + 4], coords[7 * (size_t)i + 5], coords[7 * (size_t)i + 6]);
	bool empty = false;
	map_one(ops, n_ops, pw, dw, empty);
	coords[7 * (size_t)i] = pw.x; coords[7 * (size_t)i + 1] = pw.y; coords[7 * (size_t)i + 2] = pw.z;
	coords[7 * (size_t)i + 4] = dw.x; coords[7 * (size_t)i + 5] = dw.y; coords[7 * (size_t)i + 6] = dw.z;
	if (empty) empty_mask[i] = 1;
}

// EditOperator::compute_poisson_full_residuals: outputs are written only where an operator's tet contains the sample (the caller clears, :2863-2866)
__global__ void k_poisson(const DevOp* __restrict__ ops, int n_ops, const float* __restrict__ coords, uint32_t n, float* __restrict__ sh,
                          float* __restrict__ od, float* __restrict__ rd) {
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	Membrane mem;
	poisson_one(ops, n_ops, v3(coords[7 * (size_t)i], coords[7 * (size_t)i + 1], coords[7 * (size_t)i + 2]), mem);
	if (mem.op < 0) return;
	od[i] = mem.dob;
	rd[i] = mem.drb;
	for (int k = 0; k < 27; ++k) sh[27 * (size_t)i + k] = membrane_sh(ops, mem, k);
}

// EditOperator::map_positions: interpolate_tet_pos (cage_deformation.cu:136-192: no direction, and the vacated-region mask does NOT look at `copy`)
// and translate_in_box_pos (affine_duplication.cu:69-90), operators [0, n_ops) in reverse order; positions are `stride` floats apart
__global__ void k_map_positions(const DevOp* __restrict__ ops, int n_ops, float* __restrict__ pos, uint32_t stride, uint8_t* __restrict__ empty_mask, uint32_t n) {
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	float* q = pos + (size_t)i * stride;
	V3 pw = v3(q[0], q[1], q[2]);
	bool empty = false;
	for (int o = n_ops - 1; o >= 0; --o) {
		const DevOp& op = ops[o];
		if (op.type == 0) {
			if (op.n_tets == 0) continue;
			bool in_deformed = false;
			if (box_contains(op.wbmin, op.wbmax, pw)) {
				V3 p = unwarp_position(pw, op.amin, op.amax);
				float b[4];
				int t = find_tet(op, p, b);
				if (t >= 0) {
					uint4 tv = __ldg(reinterpret_cast<const uint4*>(op.tets) + t);
					pw = warp_position(bary_mix(b, ldv(op.orig_verts, tv.x), ldv(op.orig_verts, tv.y), ldv(op.orig_verts, tv.z), ldv(op.orig_verts, tv.w)), op.amin, op.amax);
					in_deformed = true;
				}
			}
			if (!in_deformed && box_contains(op.owbmin, op.owbmax, pw)) {
				V3 p = unwarp_position(pw, op.amin, op.amax);
				int level = mip_from_pos(p);
				if (bitfield_at(cascaded_grid_idx_at(p, (uint32_t)level), (uint32_t)level, op.obits)) empty = true;
			}
		} else {
			V3 dw = v3(0.5f, 0.5f, 0.5f);
			DevOp tmp_free = op;  // translate_in_box_pos never touches a direction
			tmp_free.correct_dir = 0;
			affine_map(tmp_free, pw, dw, empty);
		}
	}
	q[0] = pw.x; q[1] = pw.y; q[2] = pw.z;
	if (empty && empty_mask) empty_mask[i] = 1;
}

// The loop of compute_poisson_residual_density_kernel (cage_deformation.cu:341-383): h += (half) interpolated residual density, for the
// first tet that contains the (warped) position pw, of each operator in reverse order. Only the residual density array is required (:647-672).
__device__ __forceinline__ void add_residual_density(const DevOp* __restrict__ ops, int n_ops, V3 pw, __half& h) {
	for (int o = n_ops - 1; o >= 0; --o) {
		const DevOp& op = ops[o];
		if (op.type != 0 || !op.apply_poisson || !op.rd || op.n_tets == 0) continue;
		V3 p = unwarp_position(pw, op.amin, op.amax);
		if (!box_contains(op.bmin, op.bmax, p)) continue;
		float b[4];
		int t = find_tet(op, p, b);
		if (t < 0) continue;
		uint4 tv = __ldg(reinterpret_cast<const uint4*>(op.tets) + t);
		float res = bary_mix1(b, __ldg(op.rd + tv.x), __ldg(op.rd + tv.y), __ldg(op.rd + tv.z), __ldg(op.rd + tv.w));
		h = __hadd(h, __float2half_rn(res));
	}
}

// EditOperator::compute_poisson_residual_density: density_network_output[i] += the residual densities at position i
__global__ void k_poisson_residual_density(const DevOp* __restrict__ ops, int n_ops, const float* __restrict__ pos, uint32_t stride, __half* __restrict__ density_out, uint32_t n) {
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const float* q = pos + (size_t)i * stride;
	add_residual_density(ops, n_ops, v3(q[0], q[1], q[2]), density_out[i]);
}

template <bool GENERAL>
__global__ void k_march_trace(const DevFrame f, const uint8_t* __restrict__ bitfield, const uint32_t* __restrict__ pixels, uint32_t n_pixels,
                              uint32_t max_samples, float* __restrict__ rec, uint32_t* __restrict__ idx, uint32_t* __restrict__ count) {
	__shared__ uint32_t spread7[128];
	fill_spread7(spread7);
	__syncthreads();
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_pixels) return;
	uint32_t pix = pixels[i];
	uint32_t px = pix % (uint32_t)f.W, py = pix / (uint32_t)f.W;
	Ray r;
	uint32_t c = 0;
	if (GENERAL ? make_ray_general(f, px, py, r) : make_ray(f, px, py, r)) {
		V3 idir = v3(__frcp_rn(r.d.x), __frcp_rn(r.d.y), __frcp_rn(r.d.z));
		float t = fma_(ld_random_val(f.spp, pix * 786433u), calc_dt(r.t, f.cone), r.t);
		while (c < MARCH_ITER) {
			float dt; V3 pos; uint32_t mip, cell;
			if (!next_occupied(f, bitfield, spread7, r.o, r.d, idir, t, dt, pos, mip, cell)) break;
			if (c < max_samples) {
				float* rr = rec + ((size_t)i * max_samples + c) * 5;
				rr[0] = t; rr[1] = dt; rr[2] = pos.x; rr[3] = pos.y; rr[4] = pos.z;
				uint32_t* ii = idx + ((size_t)i * max_samples + c) * 2;
				ii[0] = mip; ii[1] = cell;
			}
			++c;
			t = add(t, dt);
		}
	}
	count[i] = c;
}

// ---- density grid -> occupancy bitfield (testbed_nerf.cu:514-555, :3642-3658) -----------------------------------------
__global__ void k_grid_mean_partial(const float* __restrict__ grid, uint32_t n, double* __restrict__ partial) {
	// fixed-shape tree: 256 threads x 64 values each per block, pairwise in shared memory (deterministic order)
	__shared__ double sh[256];
	uint32_t base = blockIdx.x * 256u * 64u + threadIdx.x * 64u;
	double acc = 0.0;
	for (uint32_t k = 0; k < 64; ++k) { uint32_t i = base + k; if (i < n) acc += (double)fmaxf(grid[i], 0.0f); }
	sh[threadIdx.x] = acc;
	__syncthreads();
	for (int s = 128; s > 0; s >>= 1) { if ((int)threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s]; __syncthreads(); }
	if (threadIdx.x == 0) partial[blockIdx.x] = sh[0];
}
__device__ __forceinline__ uint32_t morton3D_invert(uint32_t x) {
	x = x & 0x49249249u;
	x = (x | (x >> 2)) & 0xc30c30c3u;
	x = (x | (x >> 4)) & 0x0f00f00fu;
	x = (x | (x >> 8)) & 0xff0000ffu;
	x = (x | (x >> 16)) & 0x0000ffffu;
	return x;
}
__global__ void k_bitfield_max_pool(uint32_t n, const uint8_t* __restrict__ prev_level, uint8_t* __restrict__ next_level) {
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	uint8_t b = 0;
#pragma unroll
	for (int j = 0; j < 8; ++j) b |= prev_level[(size_t)i * 8 + j] > 0 ? (uint8_t)(1u << j) : (uint8_t)0;
	uint32_t x = morton3D_invert(i >> 0) + GRIDSIZE / 8, y = morton3D_invert(i >> 1) + GRIDSIZE / 8, z = morton3D_invert(i >> 2) + GRIDSIZE / 8;
	next_level[morton3D(x, y, z)] |= b;
}

// ---- occupancy update through the edit operators (testbed_nerf.cu:3533-3639) ------------------------------------------
// One fused pass per grid sample: draw (common_nerf.cu:179-208) -> map_positions in reverse operator order (:3593-3599)
// -> hash encode + density MLP on wgmma (NerfNetwork::density) -> activate (:3522-3531) -> membrane residual density
// (cage_deformation.cu:341-383) -> max-splat (:447-463). The reference materialises positions, indices, a bool mask and the
// 16 x N fp16 density matrix between seven launches; here a sample lives in registers and shared memory from draw to splat.
// It keeps its own copy of network_tiles' loop: written on network_tiles, the same code compiles to a longer hash-grid gather loop
// and runs slower.
struct GridUpdateArgs {
	uint32_t n_uniform, n_total, n_cascades, step;
	uint64_t rng_state, rng_inc;
	float amin[3], amax[3];
	int density_activation, apply_ops;
};
template <bool ACC16>
__global__ void __launch_bounds__(128) k_density_grid_update(const DevModel m, const DevOp* __restrict__ ops, int n_ops, const GridUpdateArgs a,
                                                             const float* __restrict__ grid, float* __restrict__ grid_tmp) {
	extern __shared__ __align__(128) uint8_t smem_raw[];
	tc::TileSmem& S = *reinterpret_cast<tc::TileSmem*>(smem_raw);
	const uint32_t tid = threadIdx.x;
	tc::tile_setup(S, m.w_image);
	const uint32_t n_padded = ((a.n_total + 127u) / 128u) * 128u;
	for (uint32_t base = blockIdx.x * 128u; base < n_padded; base += gridDim.x * 128u) {
		const uint32_t i = base + tid;
		const bool valid = i < a.n_total;
		V3 pw = v3(0, 0, 0), dw = v3(0.5f, 0.5f, 0.5f);
		uint32_t idx = 0;
		if (valid) {
			// the reference runs two launches (uniform: any trained cell; non-uniform: occupied cells), m_rng advanced by 2^32 between
			const bool second = i >= a.n_uniform;
			uint32_t li = second ? i - a.n_uniform : i;
			const uint32_t n_el = second ? a.n_total - a.n_uniform : a.n_uniform;
			const float thresh = second ? 0.01f : -0.01f;
			// Work assignment (not semantics): the reference's thread li draws cell (li*A + B) mod 128^3, a pseudo-random permutation,
			// so a warp's 32 samples scatter over the whole volume. Every sample is independent and the splat is an order-free max, so
			// thread t instead takes the sample whose first-choice cell is t mod 128^3: a warp covers a 4x4x2 Morton block of cells and
			// its hash-grid gathers share sectors (53369 = 56924617^-1 mod 2^21). Only whole 128^3 blocks of a launch are permuted, each within
			// itself, and a ragged tail keeps the reference's assignment, so every launch draws the reference's set of samples at any count.
			if (li < (n_el & ~(GRIDVOL - 1u)))
				li = (li & ~(GRIDVOL - 1u)) | ((((li & (GRIDVOL - 1u)) - 96925573u) * 53369u - a.step * n_el) & (GRIDVOL - 1u));
			Pcg32 rng;
			rng.state = a.rng_state; rng.inc = a.rng_inc;
			if (second) rng.advance(1ull << 32);
			rng.advance((uint64_t)(li * 4u));
			const uint32_t level = (uint32_t)mul(rng.next_float(), (float)a.n_cascades) % a.n_cascades;
			for (uint32_t j = 0; j < 10; ++j) {
				idx = ((li + a.step * n_el) * 56924617u + j * 19349663u + 96925573u) % GRIDVOL;
				idx += level * GRIDVOL;
				if (grid[idx] > thresh) break;
			}
			const uint32_t pos_idx = idx % GRIDVOL;
			const float x = (float)morton3D_invert(pos_idx >> 0), y = (float)morton3D_invert(pos_idx >> 1), z = (float)morton3D_invert(pos_idx >> 2);
			const float rx = rng.next_float(), ry = rng.next_float(), rz = rng.next_float();
			const float sc = __uint_as_float((127u + level) << 23);  // scalbnf(1, level)
			V3 p = v3(fma_(sub(div_(add(x, rx), (float)GRIDSIZE), 0.5f), sc, 0.5f), fma_(sub(div_(add(y, ry), (float)GRIDSIZE), 0.5f), sc, 0.5f),
			          fma_(sub(div_(add(z, rz), (float)GRIDSIZE), 0.5f), sc, 0.5f));
			pw = warp_position(p, a.amin, a.amax);
			if (a.apply_ops && n_ops > 0) {
				bool empty = false;  // the reference fills empty_mask here but its consumer clear_empty_space is a no-op (:2759-2770)
				V3 d = dw;
				map_one(ops, n_ops, pw, d, empty);
			}
		}
		uint32_t dens[8], rgbo[8];
		encode_to_a32(S.a32, m, valid, pw, tid);
		tc::run_network<ACC16>(tc::single_tile_ctx(S), dw, true, dens, rgbo);
		if (valid) {
			__half h = __float2half_rn(network_to_density(__half2float(__ushort_as_half((unsigned short)(dens[0] & 0xffffu))), a.density_activation));
			if (a.apply_ops) add_residual_density(ops, n_ops, pw, h);  // :3612-3620; looked up at the MAPPED position, as the reference does
			const float optical_thickness = mul(__half2float(h), MIN_STEP());
			atomicMax(reinterpret_cast<unsigned int*>(grid_tmp) + idx, __float_as_uint(optical_thickness));  // uint order == float order for >= 0
		}
	}
}
__global__ void k_ema_grid(uint32_t n, float decay, float* __restrict__ grid, const float* __restrict__ grid_tmp) {  // :483-506
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	float prev = grid[i];
	grid[i] = prev < 0.0f ? prev : fmaxf(mul(prev, decay), grid_tmp[i]);
}
__global__ void k_grid_mean_final(const double* __restrict__ partial, uint32_t n_blocks, uint32_t n0, float* __restrict__ thresh_out) {
	double sum = 0.0;
	for (uint32_t k = 0; k < n_blocks; ++k) sum += partial[k];  // fixed order
	const float mean = (float)(sum / (double)n0);
	thresh_out[0] = mean < 0.01f ? mean : 0.01f;  // std::min(NERF_MIN_OPTICAL_THICKNESS(), mean) (:524)
	thresh_out[1] = mean;
}
__global__ void k_grid_to_bitfield_dev(uint32_t n_bytes, const float* __restrict__ grid, uint8_t* __restrict__ bits, const float* __restrict__ thresh_ptr) {
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_bytes) return;
	const float thresh = thresh_ptr[0];
	uint8_t b = 0;
#pragma unroll
	for (int j = 0; j < 8; ++j) b |= grid[(size_t)i * 8 + j] > thresh ? (uint8_t)(1u << j) : (uint8_t)0;
	bits[i] = b;
}

// ---- frame post-process: accumulate_kernel (render_buffer.cu:217-258) and tonemap_kernel (:471-499) -------------------
__device__ __forceinline__ float linear_to_srgb(float l) {  // common_device.cuh:53-59
	if (l < 0.0031308f) return 12.92f * l;
	return 1.055f * powf(l, 0.41666f) - 0.055f;
}
__global__ void k_accumulate(int n, const float4* __restrict__ frame, float4* __restrict__ acc, float sample_count, int color_space) {
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	float4 c = frame[i], t = acc[i];
	const float inv = sample_count + 1.0f;
	if (color_space == NSB_COLOR_VISPOSNEG) {
		float val = c.x - c.y, tmp_val = t.x - t.y;
		tmp_val = (tmp_val * sample_count + val) / inv;
		t.x = fmaxf(tmp_val, 0.0f);
		t.y = fmaxf(-tmp_val, 0.0f);
	} else {
		if (color_space == NSB_COLOR_SRGB) { c.x = linear_to_srgb(c.x); c.y = linear_to_srgb(c.y); c.z = linear_to_srgb(c.z); }
		t.x = (t.x * sample_count + c.x) / inv;
		t.y = (t.y * sample_count + c.y) / inv;
		t.z = (t.z * sample_count + c.z) / inv;
	}
	t.w = (t.w * sample_count + c.w) / inv;
	acc[i] = t;
}
__device__ __forceinline__ void tonemap_curve(float* x, int curve) {  // render_buffer.cu:262-310
	if (curve == NSB_TONEMAP_IDENTITY) return;
	for (int k = 0; k < 3; ++k) x[k] = fmaxf(x[k], 0.0f);
	float k0, k1, k2, k3, k4, k5;
	if (curve == NSB_TONEMAP_ACES) {
		k0 = 0.6f * 0.6f * 2.51f; k1 = 0.6f * 0.03f; k2 = 0.0f; k3 = 0.6f * 0.6f * 2.43f; k4 = 0.6f * 0.59f; k5 = 0.14f;
	} else if (curve == NSB_TONEMAP_HABLE) {
		const float A = 0.15f, B = 0.50f, C = 0.10f, D = 0.20f, E = 0.02f, F = 0.30f;
		k0 = A * F - A * E; k1 = C * B * F - B * E; k2 = 0.0f; k3 = A * F; k4 = B * F; k5 = D * F * F;
		const float W = 11.2f;
		const float nom = k0 * (W * W) + k1 * W + k2, denom = k3 * (W * W) + k4 * W + k5;
		const float white_scale = denom / nom;
		k0 = 4.0f * k0 * white_scale; k1 = 2.0f * k1 * white_scale; k2 = k2 * white_scale; k3 = 4.0f * k3; k4 = 2.0f * k4;
	} else {  // Reinhard
		// luminance_coefficients.dot(x): Eigen reduces a 3-vector as x0 + (x1 + x2), which nvcc contracts into these two FMAs
		float Y = __fmaf_rn(0.2126f, x[0], __fmaf_rn(0.7152f, x[1], __fmul_rn(0.0722f, x[2])));
		float s = 1.0f / (Y + 1.0f);
		for (int k = 0; k < 3; ++k) x[k] *= s;
		return;
	}
	for (int k = 0; k < 3; ++k) {  // color_sq * k0 + k1 * x + k2 and k3 * color_sq + k4 * x + k5 as nvcc contracts them in the reference
		const float sq = __fmul_rn(x[k], x[k]);
		const float nom = __fadd_rn(__fmaf_rn(sq, k0, __fmul_rn(k1, x[k])), k2);
		const float denom = __fadd_rn(__fmaf_rn(k3, sq, __fmul_rn(k4, x[k])), k5);
		x[k] = nom / denom;
	}
}
__global__ void k_tonemap(int n, const float4* __restrict__ acc, float4* __restrict__ out, NsbTonemap p) {
	int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	float bg[4] = {p.background_color[0], p.background_color[1], p.background_color[2], p.background_color[3]};
	if (p.color_space != NSB_COLOR_SRGB) for (int k = 0; k < 3; ++k) bg[k] = srgb_to_linear(bg[k]);
	float4 c4 = acc[i];
	float c[3] = {c4.x, c4.y, c4.z};
	float weight = (1.0f - c4.w) * bg[3];
	for (int k = 0; k < 3; ++k) c[k] += bg[k] * weight;
	float a = c4.w + weight;
	if (p.color_space == NSB_COLOR_SRGB) for (int k = 0; k < 3; ++k) c[k] = srgb_to_linear(c[k]);
	const float e = powf(2.0f, p.exposure);
	for (int k = 0; k < 3; ++k) c[k] *= e;
	tonemap_curve(c, p.tonemap_curve);
	if (p.output_color_space == NSB_COLOR_SRGB) for (int k = 0; k < 3; ++k) c[k] = linear_to_srgb(c[k]);
	if (p.clamp_output_color) { for (int k = 0; k < 3; ++k) c[k] = fminf(fmaxf(c[k], 0.0f), 1.0f); a = fminf(fmaxf(a, 0.0f), 1.0f); }
	out[i] = make_float4(c[0], c[1], c[2], a);
}

// packed tile buffers for the single multi-GPU framebuffer gather
__global__ void k_pack_tiles(const float4* __restrict__ fb, const float* __restrict__ depth, int W, int H, int tiles_x, int n_tiles, int rank, int world,
                             float4* __restrict__ dst, float* __restrict__ dst_depth, int unpack) {
	uint32_t local = blockIdx.x;
	uint32_t tile = (uint32_t)rank + local * (uint32_t)world;
	if (tile >= (uint32_t)n_tiles) return;
	uint32_t lane = threadIdx.x;  // 0..127
	uint32_t px = (tile % (uint32_t)tiles_x) * TILE_W + (lane % TILE_W), py = (tile / (uint32_t)tiles_x) * TILE_H + (lane / TILE_W);
	if (px >= (uint32_t)W || py >= (uint32_t)H) return;
	size_t p = (size_t)px + (size_t)W * py, q = (size_t)local * TILE_PIXELS + lane;
	if (!unpack) {
		dst[q] = fb[p];
		if (dst_depth && depth) dst_depth[q] = depth[p];
	} else {
		const_cast<float4*>(fb)[p] = dst[q];
		if (dst_depth && depth) const_cast<float*>(depth)[p] = dst_depth[q];
	}
}

// all the OTHER ranks' shards of one all-gather -> the framebuffer (and depth), ONE launch: block = (local tile, source rank)
__global__ void k_unpack_gathered(const float4* __restrict__ gathered, const float* __restrict__ gathered_depth, int W, int H, int tiles_x, int n_tiles, int skip_rank,
                                  int world, uint32_t rank_stride /*floats between two ranks' shards, in BOTH arrays*/, float4* __restrict__ fb, float* __restrict__ depth) {
	const uint32_t local = blockIdx.x, rank = blockIdx.y;
	if ((int)rank == skip_rank) return;
	const uint32_t tile = rank + local * (uint32_t)world;
	if (tile >= (uint32_t)n_tiles) return;
	const uint32_t lane = threadIdx.x;
	const uint32_t px = (tile % (uint32_t)tiles_x) * TILE_W + (lane % TILE_W), py = (tile / (uint32_t)tiles_x) * TILE_H + (lane / TILE_W);
	if (px >= (uint32_t)W || py >= (uint32_t)H) return;
	const size_t p = (size_t)px + (size_t)W * py, q = (size_t)local * TILE_PIXELS + lane;
	fb[p] = gathered[(size_t)rank * (rank_stride / 4) + q];
	if (depth && gathered_depth) depth[p] = gathered_depth[(size_t)rank * rank_stride + q];
}

#include "nsb_mesh.cuh"
#include "nsb_mesh_opt.cuh"
#include "nsb_slices.cuh"
#include "nsb_video.cuh"

// =====================================================================================================
// host side: context, uploads, C ABI
// =====================================================================================================
#include "nsb_edit_rebuild.cuh"
static thread_local std::string g_last_error;
static NsbStatus fail(NsbStatus s, const char* fmt, ...) {
	char buf[512];
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(buf, sizeof(buf), fmt, ap);
	va_end(ap);
	g_last_error = buf;
	return s;
}
#define CU(call)                                                                                                 \
	do {                                                                                                         \
		cudaError_t e__ = (call);                                                                                \
		if (e__ != cudaSuccess) return fail(NSB_ERR_CUDA, "%s: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, __LINE__); \
	} while (0)

// Owner of one device array of T. reserve() only grows and does not keep the contents. A failed reserve leaves the buffer empty
// (null, capacity 0), so a buffer never reports room it does not have.
template <typename T>
class DevBuf {
	T* p_ = nullptr;
	size_t n_ = 0;  // capacity in elements

public:
	DevBuf() = default;
	DevBuf(DevBuf&& o) noexcept : p_(o.p_), n_(o.n_) { o.p_ = nullptr; o.n_ = 0; }
	DevBuf& operator=(DevBuf&& o) noexcept { std::swap(p_, o.p_); std::swap(n_, o.n_); return *this; }  // the old array goes with o
	~DevBuf() { cudaFree(p_); }
	cudaError_t reserve(size_t n) {
		if (n <= n_) return cudaSuccess;
		cudaFree(p_);
		n_ = 0;
		const cudaError_t e = cudaMalloc(&p_, n * sizeof(T));
		if (e == cudaSuccess) n_ = n;
		else p_ = nullptr;
		return e;
	}
	T* get() const { return p_; }
	size_t capacity() const { return n_; }
};

struct NsbContext {
	int device = 0;
	int sm_count = 0;
	int inference_ctas_per_sm = 1;
	int grid_update_ctas_per_sm = 1;
	bool has_model = false, has_occ = false;
	NsbModelDesc desc{};
	DevModel model{};
	bool dense_in_range = false;       // the model's dense levels admit grid_index's in-range shortcut (nsb_device.cuh)
	DevBuf<__half2> d_grid;
	DevBuf<uint8_t> d_wimage;
	DevBuf<__half> d_wrow;
	DevBuf<uint8_t> d_bitfield;
	DevBuf<float> d_density_grid;      // running density grid, 5 x 128^3 (Testbed::Nerf::density_grid, testbed.h:622)
	DevBuf<float> d_density_tmp;       // density_grid_tmp scratch of an update
	DevBuf<double> d_mean_partial;
	DevBuf<float> d_thresh;            // [0] bitfield threshold, [1] mean of cascade 0
	DevBuf<DevOp> d_ops;
	int n_ops = 0;
	int any_poisson = 0;
	std::vector<DevOp> h_ops;          // host copy of d_ops (pointers are device pointers)
	struct CageArrays {                // device arrays of one operator slot (empty for an affine operator)
		// what the slot's DevOp points at, as uploaded by nsb_set_edit_ops; nsb_cage_deform rewrites verts/rots/lut_* in place
		DevBuf<uint32_t> lut_off, lut_idx, tets;
		DevBuf<float> verts, orig_verts, rots, shs, od, rd;
		DevBuf<uint8_t> obits;
		uint32_t n_vertices = 0;
		uint64_t n_idx = 0;            // entries of lut_idx in use
		// nsb_cage_attach_mvc / nsb_cage_deform
		DevBuf<float> d_mvc; uint32_t n_cv = 0;
		DevBuf<float> d_cage;
		DevBuf<uint32_t> d_counts, d_block_sums, d_total;
		DevBuf<nsb::rebuild::Mark> d_marks; DevBuf<unsigned int> d_n_marks;
		DevBuf<float> d_boxes;         // [12] bbox min/max, warped min/max; [12..17] scene aabb
		DevBuf<float> d_gamma, d_mem_small;  // nsb_cage_set_membrane scratch
	};
	std::vector<CageArrays> rb;
	DevBuf<uint32_t> d_counters;       // [0] rays queued by k_prepare_rays, [1] fetch cursor of k_render_fused
	DevBuf<unsigned long long> d_n_cleared;  // cells a counted nsb_cage_vanish changed
	DevBuf<unsigned long long> d_stats;
	DevBuf<RayRec> d_list;
	DevBuf<float> d_ray_od;            // origin + direction per queue slot, general-camera frames only (allocated on the first such frame)
	int acc16 = 1;                 // MLP accumulator policy: 1 fp16 wgmma accumulators (default: the reference's wmma __half fragments), 0 fp32 (nsb_set_mlp_accumulator)
	cudaEvent_t ev0 = nullptr, ev1 = nullptr, evm = nullptr;  // start, end, between k_prepare_rays and k_render_fused
	bool timed = false;
	uint32_t launches = 0;
	DevBuf<float> d_fb, d_depth;       // nsb_render_host
	DevBuf<float> d_sub_fb, d_sub_depth;  // nsb_render_accumulate: the frame and depth buffers each sub-frame is rendered into
	cudaStream_t stream = nullptr;
	// nsb_render_host_async: two framebuffers in flight, the D2H copy of one overlaps the render of the other
	DevBuf<float> d_fb2[2], d_depth2[2];
	cudaStream_t copy_stream = nullptr;
	cudaEvent_t render_done[2] = {nullptr, nullptr}, copy_done[2] = {nullptr, nullptr};
	uint64_t host_seq = 0;  // tickets issued
	// the mesh of nsb_marching_cubes (Testbed::m_mesh): vertex rows = n_vertices rounded up to 128 like marching_cubes.cu:751-753, the padding
	// rows at the origin; normals and colours are written by nsb_mesh_shade
	DevBuf<float> mesh_verts, mesh_normals, mesh_colors;
	DevBuf<uint32_t> mesh_idx;
	uint64_t mesh_nv = 0, mesh_ni = 0;
	bool has_mesh = false, mesh_shaded = false;
	DevBuf<uint32_t> mc_voff, mc_tiles;  // first vertex id per grid point (4 B per point), per-tile vertex and triangle offsets
	DevBuf<unsigned long long> mc_totals;
	DevBuf<uint32_t> mesh_start, mesh_cursor, mesh_adj;  // per-vertex triangle lists (CSR) of nsb_mesh_shade and nsb_mesh_optimise
	DevBuf<uint8_t> mesh_scan_tmp;
	bool mesh_csr = false;      // mesh_start / mesh_adj describe the current mesh
	bool mesh_normals_ok = false;  // mesh_normals describe the current mesh (nsb_mesh_shade, nsb_mesh_optimise)
	// nsb_mesh_optimise: Adam state per vertex row (moments, step counters: 36 B) and the ping-pong position buffer (12 B), allocated on the
	// first call and reset by the first call after each nsb_marching_cubes; density (2 B) and position gradient (12 B) of the current step
	DevBuf<float> opt_pos, opt_m1, opt_m2, opt_grad;
	DevBuf<uint32_t> opt_steps;
	DevBuf<__half> opt_dens;
	bool opt_fresh = true;

	~NsbContext() {  // the device arrays free themselves
		for (cudaEvent_t e : {ev0, ev1, evm, render_done[0], render_done[1], copy_done[0], copy_done[1]}) if (e) cudaEventDestroy(e);
		for (cudaStream_t s : {stream, copy_stream}) if (s) cudaStreamDestroy(s);
	}
};

static uint32_t next_multiple_u32(uint32_t v, uint32_t m) { return ((v + m - 1) / m) * m; }

// The grid of a one-tile kernel over n_rows rows: one 128-row tile per CTA, at most ctas_per_sm resident CTAs per SM (the kernels
// stride over the rest)
static uint32_t tile_ctas(const NsbContext* c, uint64_t n_rows, int ctas_per_sm) {
	const uint64_t tiles = (n_rows + 127) / 128, cap = (uint64_t)c->sm_count * ctas_per_sm;
	return (uint32_t)(tiles < cap ? tiles : cap);
}

static const uint64_t kMlpParams = 64 * 32 + 16 * 64 + 64 * 32 + 64 * 64 + 16 * 64;

extern "C" int nsb_abi_version(void) { return NSB_ABI_VERSION; }
extern "C" const char* nsb_last_error(void) { return g_last_error.c_str(); }

extern "C" NsbStatus nsb_model_n_params(const NsbModelDesc* desc, uint64_t* n_params) {
	DevLevel L[MAX_LEVELS];
	uint64_t n = 0;
	if (!n_params || !build_levels(desc, L, &n)) return fail(NSB_ERR_INVALID, "unsupported model description (only the configs/nerf/base.json topology is implemented)");
	*n_params = kMlpParams + 2 * n;
	return NSB_OK;
}

extern "C" NsbStatus nsb_create(int device, NsbContext** out) {
	if (!out) return fail(NSB_ERR_INVALID, "out is null");
	int n_dev = 0;
	CU(cudaGetDeviceCount(&n_dev));
	if (n_dev == 0) return fail(NSB_ERR_CUDA, "no CUDA device: nerfshop_b200 has no CPU fallback");
	if (device < 0) CU(cudaGetDevice(&device));
	if (device >= n_dev) return fail(NSB_ERR_INVALID, "device %d out of range (%d devices)", device, n_dev);
	CU(cudaSetDevice(device));
	cudaDeviceProp prop;
	CU(cudaGetDeviceProperties(&prop, device));
	if (prop.major != 9 || prop.minor != 0) return fail(NSB_ERR_UNSUPPORTED, "device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, prop.major, prop.minor);
	std::unique_ptr<NsbContext> c(new NsbContext());  // released to the caller only once complete
	c->device = device;
	c->sm_count = prop.multiProcessorCount;
	CU(c->d_counters.reserve(2));
	CU(c->d_n_cleared.reserve(1));
	CU(c->d_stats.reserve(ST_N));
	CU(cudaMemset(c->d_stats.get(), 0, ST_N * sizeof(unsigned long long)));
	CU(cudaEventCreate(&c->ev0));
	CU(cudaEventCreate(&c->ev1));
	CU(cudaEventCreate(&c->evm));
	CU(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
	CU(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
	for (int i = 0; i < 2; ++i) {
		CU(cudaEventCreateWithFlags(&c->render_done[i], cudaEventDisableTiming));
		CU(cudaEventCreateWithFlags(&c->copy_done[i], cudaEventDisableTiming));
	}
	// Shared memory and L1 share one 256 KB array per SM: every kernel asks for exactly the carve-out its resident CTAs need and
	// leaves the rest to L1, which serves the hash-grid gathers (the default heuristic picks a carve-out too small for even one
	// CTA; "max shared" starves L1).
	auto set_smem = [&](const void* func, size_t bytes_per_cta, int ctas) -> cudaError_t {
		cudaError_t e = cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes_per_cta);
		if (e != cudaSuccess) return e;
		const size_t need = (bytes_per_cta + 1024) * (size_t)ctas;  // 1 KB per CTA is reserved by the system
		int pct = (int)((need * 100 + prop.sharedMemPerMultiprocessor - 1) / prop.sharedMemPerMultiprocessor);
		if (pct > 100) pct = 100;
		return cudaFuncSetAttribute(func, cudaFuncAttributePreferredSharedMemoryCarveout, pct);
	};
	// k_render_fused: ONE CTA of render_tiles(OPS, ACC16) tiles per SM (896 x 72 / 768 x 80 / 640 x 96 registers = the register file;
	// shared memory 20 KB weights + 14.5 KB per tile).
	CU(set_smem((const void*)k_render_fused<false, false, true>, sizeof(RenderSmemT<render_tiles(false, false)>), 1));
	CU(set_smem((const void*)k_render_fused<false, true, true>, sizeof(RenderSmemT<render_tiles(false, true)>), 1));
	CU(set_smem((const void*)k_render_fused<false, false, false>, sizeof(RenderSmemT<render_tiles(false, false)>), 1));
	CU(set_smem((const void*)k_render_fused<false, true, false>, sizeof(RenderSmemT<render_tiles(false, true)>), 1));
	CU(set_smem((const void*)k_render_fused<true, false, false>, sizeof(RenderSmemT<render_tiles(true, false)>), 1));
	CU(set_smem((const void*)k_render_fused<true, true, false>, sizeof(RenderSmemT<render_tiles(true, true)>), 1));
	cudaFuncAttributes fa;
	CU(cudaFuncGetAttributes(&fa, k_render_fused<false, true, true>));
	// the operator-level kernels: one tile per CTA, residency from registers / shared memory, 1 to 5 CTAs per SM
	auto tile_ctas_per_sm = [&](const void* func, int* ctas) -> cudaError_t {
		cudaFuncAttributes fi;
		const cudaError_t e = cudaFuncGetAttributes(&fi, func);
		if (e != cudaSuccess) return e;
		const int by_regs = fi.numRegs > 0 ? (int)(prop.regsPerMultiprocessor / (fi.numRegs * 128)) : 4;
		const int by_smem = (int)(prop.sharedMemPerMultiprocessor / (sizeof(tc::TileSmem) + 1024));
		const int r = by_regs < by_smem ? by_regs : by_smem;
		*ctas = r > 5 ? 5 : r < 1 ? 1 : r;
		return cudaSuccess;
	};
	CU(tile_ctas_per_sm((const void*)k_inference<false, false>, &c->inference_ctas_per_sm));
	CU(tile_ctas_per_sm((const void*)k_density_grid_update<false>, &c->grid_update_ctas_per_sm));
	for (const void* f : {(const void*)k_inference<false, false>, (const void*)k_inference<true, false>, (const void*)k_inference<false, true>,
	                      (const void*)k_inference<true, true>, (const void*)mesh::k_density_on_grid<false>, (const void*)mesh::k_density_on_grid<true>,
	                      (const void*)mesh::k_mesh_colors<false>, (const void*)mesh::k_mesh_colors<true>, (const void*)slices::k_rgba_on_grid<false>,
	                      (const void*)slices::k_rgba_on_grid<true>})
		CU(set_smem(f, sizeof(tc::TileSmem), c->inference_ctas_per_sm));
	for (const void* f : {(const void*)k_density_grid_update<false>, (const void*)k_density_grid_update<true>})
		CU(set_smem(f, sizeof(tc::TileSmem), c->grid_update_ctas_per_sm));
	for (const void* f : {(const void*)meshopt::k_density_gradient<false, false>, (const void*)meshopt::k_density_gradient<true, false>,
	                      (const void*)meshopt::k_density_gradient<false, true>, (const void*)meshopt::k_density_gradient<true, true>})
		CU(set_smem(f, sizeof(meshopt::GradSmem), c->inference_ctas_per_sm));
	if (getenv("NSB_VERBOSE"))
		fprintf(stderr, "[nsb] device %d: %d SMs; k_render_fused %d tiles/CTA (%d with fp32 accumulators, %d with operators), %d regs, %zu B smem; inference %d CTAs/SM, grid update %d CTAs/SM\n",
		        device, c->sm_count, render_tiles(false, true), render_tiles(false, false), render_tiles(true, true), fa.numRegs, sizeof(RenderSmemT<render_tiles(false, true)>),
		        c->inference_ctas_per_sm, c->grid_update_ctas_per_sm);
	*out = c.release();
	return NSB_OK;
}

extern "C" NsbStatus nsb_destroy(NsbContext* c) {
	if (!c) return NSB_OK;
	cudaSetDevice(c->device);
	cudaDeviceSynchronize();
	delete c;
	return NSB_OK;
}

// [N x K] row-major fp16 -> wgmma K-major no-swizzle operand image (nsb_tc.cuh header comment)
static void to_operand_layout(const uint16_t* W, uint32_t N, uint32_t K, uint8_t* dst) {
	for (uint32_t n = 0; n < N; ++n)
		for (uint32_t k = 0; k < K; ++k) {
			size_t off = (size_t)(k / 8) * (N * 16) + (size_t)n * 16 + (k % 8) * 2;
			memcpy(dst + off, W + (size_t)n * K + k, 2);
		}
}

// params_on_device: the block is read where tcnn::Trainer keeps it; only the 20 KB of MLP weights pass through the host (to be laid out as wgmma operands)
static NsbStatus upload_model_impl(NsbContext* c, const NsbModelDesc* desc, const uint16_t* params, uint64_t n_params, bool params_on_device) {
	if (!c || !desc || !params) return fail(NSB_ERR_INVALID, "null argument");
	CU(cudaSetDevice(c->device));
	DevModel m{};
	uint64_t n_grid = 0;
	if (!build_levels(desc, m.levels, &n_grid)) return fail(NSB_ERR_INVALID, "unsupported model description (only the configs/nerf/base.json topology is implemented)");
	if (n_params != kMlpParams + 2 * n_grid) return fail(NSB_ERR_INVALID, "n_params %llu != expected %llu", (unsigned long long)n_params, (unsigned long long)(kMlpParams + 2 * n_grid));
	CU(cudaDeviceSynchronize());
	// has_model implies that model points into live buffers: it is cleared before the old model's buffers are released, and set again
	// only once the new model is complete
	c->has_model = false;
	c->d_grid = {}; c->d_wimage = {}; c->d_wrow = {};
	// block order: density MLP, rgb MLP, hash grid (nerf_network_full.h:316-349)
	std::vector<uint8_t> image(tc::W_BYTES);
	std::vector<uint16_t> mlp_host;
	if (params_on_device) {
		mlp_host.resize(kMlpParams);
		CU(cudaMemcpy(mlp_host.data(), params, kMlpParams * 2, cudaMemcpyDeviceToHost));
	}
	const uint16_t* w = params_on_device ? mlp_host.data() : params;
	to_operand_layout(w, 64, 32, image.data() + tc::W1_OFF); w += 64 * 32;
	to_operand_layout(w, 16, 64, image.data() + tc::W2_OFF); w += 16 * 64;
	to_operand_layout(w, 64, 32, image.data() + tc::W3_OFF); w += 64 * 32;
	to_operand_layout(w, 64, 64, image.data() + tc::W4_OFF); w += 64 * 64;
	to_operand_layout(w, 16, 64, image.data() + tc::W5_OFF); w += 16 * 64;
	CU(c->d_wimage.reserve(tc::W_BYTES));
	CU(cudaMemcpy(c->d_wimage.get(), image.data(), tc::W_BYTES, cudaMemcpyHostToDevice));
	CU(c->d_wrow.reserve(kMlpParams));
	CU(cudaMemcpy(c->d_wrow.get(), params, kMlpParams * 2, params_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
	CU(c->d_grid.reserve(n_grid));
	CU(cudaMemcpy(c->d_grid.get(), params + kMlpParams, n_grid * 4, params_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
	m.grid = c->d_grid.get();
	for (uint32_t l = 0; l < desc->n_levels; ++l) m.levels[l].base = c->d_grid.get() + (uintptr_t)m.levels[l].base / sizeof(__half2);
	m.w_image = c->d_wimage.get();
	m.w_rowmajor = c->d_wrow.get();
	m.n_levels = desc->n_levels;
	for (int g = 0; g < MAX_LEVELS / 2; ++g) {
		uint32_t a = m.levels[2 * g].hashed, b = m.levels[2 * g + 1].hashed;
		m.pair_mode[g] = (a && b) ? 1u : ((!a && !b) ? 0u : 2u);
	}
	c->model = m;
	c->desc = *desc;
	c->dense_in_range = dense_in_range(m.levels, m.n_levels);
	c->has_model = true;
	return NSB_OK;
}

extern "C" NsbStatus nsb_upload_model(NsbContext* c, const NsbModelDesc* desc, const uint16_t* params, uint64_t n_params) {
	return upload_model_impl(c, desc, params, n_params, false);
}
extern "C" NsbStatus nsb_upload_model_dev(NsbContext* c, const NsbModelDesc* desc, const uint16_t* params_dev, uint64_t n_params) {
	return upload_model_impl(c, desc, params_dev, n_params, true);
}

static NsbStatus upload_occupancy_impl(NsbContext* c, const uint8_t* bitfield, uint64_t n_bytes, bool on_device) {
	if (!c || !bitfield) return fail(NSB_ERR_INVALID, "null argument");
	if (n_bytes != NSB_BITFIELD_BYTES) return fail(NSB_ERR_INVALID, "bitfield must be %u bytes (5 x 128^3 / 8)", NSB_BITFIELD_BYTES);
	CU(cudaSetDevice(c->device));
	CU(c->d_bitfield.reserve(NSB_BITFIELD_BYTES));
	CU(cudaDeviceSynchronize());
	CU(cudaMemcpy(c->d_bitfield.get(), bitfield, NSB_BITFIELD_BYTES, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
	c->has_occ = true;
	return NSB_OK;
}
extern "C" NsbStatus nsb_upload_occupancy(NsbContext* c, const uint8_t* bitfield, uint64_t n_bytes) { return upload_occupancy_impl(c, bitfield, n_bytes, false); }
extern "C" NsbStatus nsb_upload_occupancy_dev(NsbContext* c, const uint8_t* bitfield_dev, uint64_t n_bytes) { return upload_occupancy_impl(c, bitfield_dev, n_bytes, true); }

static NsbStatus ensure_grid_buffers(NsbContext* c) {
	const uint32_t n_blocks = (GRIDVOL + 256 * 64 - 1) / (256 * 64);
	if (!c->d_density_grid.get()) {  // the grid is either zeroed or not allocated: it joins the context once zeroed
		DevBuf<float> grid;
		CU(grid.reserve(NSB_GRID_CELLS));
		CU(cudaMemset(grid.get(), 0, (size_t)NSB_GRID_CELLS * 4));
		c->d_density_grid = std::move(grid);
	}
	CU(c->d_mean_partial.reserve(n_blocks));
	CU(c->d_thresh.reserve(2));
	CU(c->d_bitfield.reserve(NSB_BITFIELD_BYTES));
	return NSB_OK;
}
// Testbed::update_density_grid_mean_and_bitfield (testbed_nerf.cu:3642-3658), device-resident and stream-ordered
static NsbStatus rebuild_bitfield(NsbContext* c, cudaStream_t st) {
	const uint32_t n0 = GRIDVOL, n_blocks = (n0 + 256 * 64 - 1) / (256 * 64);
	k_grid_mean_partial<<<n_blocks, 256, 0, st>>>(c->d_density_grid.get(), n0, c->d_mean_partial.get());  // reduce_sum(fmaxf(val,0)/n) over cascade 0 (:3650)
	k_grid_mean_final<<<1, 1, 0, st>>>(c->d_mean_partial.get(), n_blocks, n0, c->d_thresh.get());
	k_grid_to_bitfield_dev<<<(NSB_BITFIELD_BYTES + 255) / 256, 256, 0, st>>>(NSB_BITFIELD_BYTES, c->d_density_grid.get(), c->d_bitfield.get(), c->d_thresh.get());
	for (uint32_t level = 1; level < NSB_NERF_CASCADES; ++level) {
		const uint32_t n = GRIDVOL / 64;
		uint8_t* bits = c->d_bitfield.get();
		k_bitfield_max_pool<<<(n + 255) / 256, 256, 0, st>>>(n, bits + (size_t)(level - 1) * (GRIDVOL / 8), bits + (size_t)level * (GRIDVOL / 8));
	}
	CU(cudaGetLastError());
	c->has_occ = true;
	return NSB_OK;
}

extern "C" NsbStatus nsb_upload_density_grid(NsbContext* c, const float* grid, uint64_t n_floats, uint8_t* bitfield_out) {
	if (!c || !grid) return fail(NSB_ERR_INVALID, "null argument");
	if (n_floats != (uint64_t)NSB_GRID_CELLS) return fail(NSB_ERR_INVALID, "density grid must be 5 x 128^3 floats");
	CU(cudaSetDevice(c->device));
	CU(cudaDeviceSynchronize());
	NsbStatus st = ensure_grid_buffers(c);
	if (st != NSB_OK) return st;
	CU(cudaMemcpy(c->d_density_grid.get(), grid, n_floats * 4, cudaMemcpyHostToDevice));
	st = rebuild_bitfield(c, nullptr);
	if (st != NSB_OK) return st;
	CU(cudaDeviceSynchronize());
	if (bitfield_out) CU(cudaMemcpy(bitfield_out, c->d_bitfield.get(), NSB_BITFIELD_BYTES, cudaMemcpyDeviceToHost));
	return NSB_OK;
}

extern "C" NsbStatus nsb_update_density_grid(NsbContext* c, const NsbGridUpdate* u, void* stream_) {
	if (!c || !u) return fail(NSB_ERR_INVALID, "null argument");
	if (!c->has_model) return fail(NSB_ERR_STATE, "nsb_upload_model has not been called");
	if (u->n_cascades < 1 || u->n_cascades > NSB_NERF_CASCADES) return fail(NSB_ERR_INVALID, "n_cascades must be in [1, 5]");
	const uint64_t n_total64 = (uint64_t)u->n_uniform_samples + u->n_nonuniform_samples;
	// k_density_grid_update's 32-bit grid-stride index must not wrap: base < 2^31 plus one stride of at most a few thousand CTAs x 128
	if (n_total64 > NSB_GRID_UPDATE_MAX_SAMPLES) return fail(NSB_ERR_INVALID, "n_uniform_samples + n_nonuniform_samples exceeds 2^31");
	CU(cudaSetDevice(c->device));
	cudaStream_t st = (cudaStream_t)stream_;
	NsbStatus rc = ensure_grid_buffers(c);
	if (rc != NSB_OK) return rc;
	CU(c->d_density_tmp.reserve(NSB_GRID_CELLS));
	if (u->reset_grid) CU(cudaMemsetAsync(c->d_density_grid.get(), 0, (size_t)NSB_GRID_CELLS * 4, st));  // :3558-3560
	CU(cudaMemsetAsync(c->d_density_tmp.get(), 0, (size_t)NSB_GRID_CELLS * 4, st));                      // :3563
	const uint32_t n_total = (uint32_t)n_total64;
	if (n_total > 0) {
		GridUpdateArgs a{};
		a.n_uniform = u->n_uniform_samples; a.n_total = n_total; a.n_cascades = (uint32_t)u->n_cascades; a.step = u->ema_step;
		a.rng_state = u->rng_state; a.rng_inc = u->rng_inc;
		for (int k = 0; k < 3; ++k) { a.amin[k] = u->train_aabb_min[k]; a.amax[k] = u->train_aabb_max[k]; }
		a.density_activation = u->density_activation; a.apply_ops = u->apply_operators ? 1 : 0;
		(c->acc16 ? k_density_grid_update<true> : k_density_grid_update<false>)<<<tile_ctas(c, n_total, c->grid_update_ctas_per_sm), 128, sizeof(tc::TileSmem), st>>>(c->model, c->d_ops.get(), c->n_ops, a, c->d_density_grid.get(), c->d_density_tmp.get());
	}
	k_ema_grid<<<(NSB_GRID_CELLS + 255) / 256, 256, 0, st>>>((uint32_t)NSB_GRID_CELLS, u->decay, c->d_density_grid.get(), c->d_density_tmp.get());  // :3634
	CU(cudaGetLastError());
	return rebuild_bitfield(c, st);                                                                      // :3639
}

extern "C" NsbStatus nsb_download_density_grid(NsbContext* c, float* grid_out, uint8_t* bitfield_out) {
	if (!c) return fail(NSB_ERR_INVALID, "null context");
	CU(cudaSetDevice(c->device));
	CU(cudaDeviceSynchronize());
	if (grid_out) {
		if (!c->d_density_grid.get()) return fail(NSB_ERR_STATE, "no density grid: call nsb_upload_density_grid or nsb_update_density_grid first");
		CU(cudaMemcpy(grid_out, c->d_density_grid.get(), (size_t)NSB_GRID_CELLS * 4, cudaMemcpyDeviceToHost));
	}
	if (bitfield_out) {
		if (!c->d_bitfield.get() || !c->has_occ) return fail(NSB_ERR_STATE, "no occupancy bitfield");
		CU(cudaMemcpy(bitfield_out, c->d_bitfield.get(), NSB_BITFIELD_BYTES, cudaMemcpyDeviceToHost));
	}
	return NSB_OK;
}

template <typename T>
static NsbStatus dev_copy(DevBuf<T>& buf, const T* host, size_t count, const T** out) {
	*out = nullptr;
	if (!host || count == 0) return NSB_OK;
	CU(buf.reserve(count));
	CU(cudaMemcpy(buf.get(), host, count * sizeof(T), cudaMemcpyHostToDevice));
	*out = buf.get();
	return NSB_OK;
}
static void cp3(float* d, const float* s) { d[0] = s[0]; d[1] = s[1]; d[2] = s[2]; }
static void cpbox(DevAffineBox& d, const NsbAffineBox& s) { cp3(d.mn, s.min); cp3(d.u, s.u); cp3(d.v, s.v); cp3(d.w, s.w); cp3(d.c, s.center); }

extern "C" NsbStatus nsb_set_edit_ops(NsbContext* c, const NsbEditOp* ops, int32_t n) {
	if (!c || n < 0 || (n > 0 && !ops)) return fail(NSB_ERR_INVALID, "bad arguments");
	CU(cudaSetDevice(c->device));
	CU(cudaDeviceSynchronize());
	// the old operators go first; the new ones are built in locals and join the context only once complete
	c->n_ops = c->any_poisson = 0;
	c->h_ops.clear();
	c->rb.clear();
	c->d_ops = {};
	if (n == 0) return NSB_OK;
	std::vector<DevOp> dev(n);
	std::vector<NsbContext::CageArrays> rb(n);
	int any_poisson = 0;
	for (int i = 0; i < n; ++i) {
		const NsbEditOp& s = ops[i];
		DevOp& d = dev[i];
		auto& r = rb[i];
		memset(&d, 0, sizeof(d));
		d.type = s.type;
		if (s.type == NSB_OP_CAGE) {
			d.copy = s.copy;
			d.apply_poisson = s.apply_poisson;
			d.amp = s.residual_amplitude;
			cp3(d.amin, s.scene_aabb_min); cp3(d.amax, s.scene_aabb_max);
			cp3(d.bmin, s.bbox_min); cp3(d.bmax, s.bbox_max);
			cp3(d.wbmin, s.warped_bbox_min); cp3(d.wbmax, s.warped_bbox_max);
			cp3(d.owbmin, s.original_warped_bbox_min); cp3(d.owbmax, s.original_warped_bbox_max);
			d.n_tets = s.n_tets;
			r.n_vertices = s.n_vertices;
			r.n_idx = s.n_lut_idx;
			if (s.n_tets) {
				if (!s.tet_lut_offsets || !s.tets || !s.vertices || !s.original_vertices || !s.original_bitfield || (s.n_lut_idx && !s.tet_lut_idx))
					return fail(NSB_ERR_INVALID, "cage operator %d: missing arrays", i);
				NsbStatus st;
				if ((st = dev_copy(r.lut_off, s.tet_lut_offsets, (size_t)NSB_GRID_CELLS + 1, &d.lut_off)) != NSB_OK) return st;
				if ((st = dev_copy(r.lut_idx, s.tet_lut_idx, (size_t)s.n_lut_idx, &d.lut_idx)) != NSB_OK) return st;
				if ((st = dev_copy(r.tets, s.tets, (size_t)4 * s.n_tets, &d.tets)) != NSB_OK) return st;
				if ((st = dev_copy(r.verts, s.vertices, (size_t)3 * s.n_vertices, &d.verts)) != NSB_OK) return st;
				if ((st = dev_copy(r.orig_verts, s.original_vertices, (size_t)3 * s.n_vertices, &d.orig_verts)) != NSB_OK) return st;
				if ((st = dev_copy(r.rots, s.local_rotations, (size_t)9 * s.n_tets, &d.rots)) != NSB_OK) return st;
				if ((st = dev_copy(r.obits, s.original_bitfield, (size_t)NSB_BITFIELD_BYTES, &d.obits)) != NSB_OK) return st;
				// each membrane array may come alone: the density-grid residual needs only boundary_residual_density (cage_deformation.cu:647-672),
				// the render's full residuals need all three (:675-716)
				if ((st = dev_copy(r.shs, s.boundary_shs, (size_t)27 * s.n_vertices, &d.shs)) != NSB_OK) return st;
				if ((st = dev_copy(r.od, s.boundary_outside_density, (size_t)s.n_vertices, &d.od)) != NSB_OK) return st;
				if ((st = dev_copy(r.rd, s.boundary_residual_density, (size_t)s.n_vertices, &d.rd)) != NSB_OK) return st;
				d.has_poisson_data = d.shs && d.od && d.rd;
				if (d.apply_poisson && d.has_poisson_data) any_poisson = 1;
			}
		} else if (s.type == NSB_OP_AFFINE) {
			cpbox(d.sel, s.selection_box);
			cpbox(d.dst, s.destination_box);
			cp3(d.translation, s.translation);
			cp3(d.scale, s.scale);
			memcpy(d.rot, s.rotation, sizeof(d.rot));
			d.hide_original = s.hide_original;
			d.correct_dir = s.correct_dir;
		} else {
			return fail(NSB_ERR_INVALID, "operator %d: unknown type %d", i, s.type);
		}
	}
	DevBuf<DevOp> d_ops;
	CU(d_ops.reserve(n));
	CU(cudaMemcpy(d_ops.get(), dev.data(), sizeof(DevOp) * n, cudaMemcpyHostToDevice));
	c->d_ops = std::move(d_ops);
	c->rb = std::move(rb);
	c->h_ops = std::move(dev);
	c->n_ops = n;
	c->any_poisson = any_poisson;
	return NSB_OK;
}

// ---- per-edit rebuild on the device (SURVEY.md §8f-1) ---------------------------------------------------------------
static NsbStatus cage_slot(NsbContext* c, int32_t op_index, const char* who) {
	if (!c) return fail(NSB_ERR_INVALID, "%s: null context", who);
	if (op_index < 0 || op_index >= c->n_ops) return fail(NSB_ERR_INVALID, "%s: operator index %d out of range (%d uploaded)", who, op_index, c->n_ops);
	if (c->h_ops[op_index].type != NSB_OP_CAGE || c->h_ops[op_index].n_tets == 0) return fail(NSB_ERR_INVALID, "%s: operator %d is not a cage with a tet mesh", who, op_index);
	return NSB_OK;
}
extern "C" NsbStatus nsb_cage_attach_mvc(NsbContext* c, int32_t op_index, const float* weights, uint32_t n_cage_vertices) {
	NsbStatus st = cage_slot(c, op_index, "nsb_cage_attach_mvc");
	if (st != NSB_OK) return st;
	if (!weights || n_cage_vertices == 0 || n_cage_vertices > 4096) return fail(NSB_ERR_INVALID, "nsb_cage_attach_mvc: bad weights / cage size");
	CU(cudaSetDevice(c->device));
	auto& r = c->rb[op_index];
	// the weights are either copied in or not allocated: the old ones go first, and the new ones join the operator once copied
	r.d_mvc = {}; r.d_cage = {};
	DevBuf<float> mvc;
	CU(mvc.reserve((size_t)r.n_vertices * n_cage_vertices));
	CU(r.d_cage.reserve((size_t)3 * n_cage_vertices));
	CU(cudaMemcpy(mvc.get(), weights, (size_t)r.n_vertices * n_cage_vertices * sizeof(float), cudaMemcpyHostToDevice));
	r.d_mvc = std::move(mvc);
	r.n_cv = n_cage_vertices;
	return NSB_OK;
}
extern "C" NsbStatus nsb_cage_deform(NsbContext* c, int32_t op_index, const float* cage_vertices, uint32_t n_cage_vertices, void* stream_) {
	using namespace nsb::rebuild;
	NsbStatus st = cage_slot(c, op_index, "nsb_cage_deform");
	if (st != NSB_OK) return st;
	auto& r = c->rb[op_index];
	if (!r.d_mvc.get()) return fail(NSB_ERR_STATE, "nsb_cage_deform: nsb_cage_attach_mvc has not been called for operator %d", op_index);
	if (!cage_vertices || n_cage_vertices != r.n_cv) return fail(NSB_ERR_INVALID, "nsb_cage_deform: expected %u cage vertices", r.n_cv);
	CU(cudaSetDevice(c->device));
	cudaStream_t s = (cudaStream_t)stream_;
	DevOp& d = c->h_ops[op_index];
	const uint32_t n_cells = (uint32_t)NSB_GRID_CELLS, n_scan_blocks = (n_cells + SCAN_TILE - 1) / SCAN_TILE;
	CU(r.d_counts.reserve(n_cells));
	CU(r.d_block_sums.reserve(n_scan_blocks));
	CU(r.d_total.reserve(1));
	CU(r.d_n_marks.reserve(1));
	if (!r.d_boxes.get()) {  // the scene aabb at [12..17] is either written or the boxes are not allocated
		DevBuf<float> boxes;
		CU(boxes.reserve(18));
		float aabb[6] = {d.amin[0], d.amin[1], d.amin[2], d.amax[0], d.amax[1], d.amax[2]};
		CU(cudaMemcpy(boxes.get() + 12, aabb, sizeof(aabb), cudaMemcpyHostToDevice));
		r.d_boxes = std::move(boxes);
	}
	CU(r.d_marks.reserve(1u << 20));
	float* d_verts = r.verts.get();
	const bool verbose = getenv("NSB_VERBOSE") != nullptr;
	auto now = [] { timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts); return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6; };
	const double t_start = now();
	double t_marked = 0, t_launched = 0;
	// 1. Cage::interpolate_with_mvc
	CU(cudaMemcpyAsync(r.d_cage.get(), cage_vertices, (size_t)3 * r.n_cv * sizeof(float), cudaMemcpyHostToDevice, s));
	k_mvc_apply<<<(r.n_vertices + 127) / 128, 128, 3 * r.n_cv * sizeof(float), s>>>(r.d_mvc.get(), r.n_vertices, r.n_cv, r.d_cage.get(), d_verts);
	// 2. TetMesh::post_update_vertices, update_local_rotations
	float* d_boxes = r.d_boxes.get();
	k_cage_bbox<<<1, 256, 0, s>>>(d_verts, r.n_vertices, d_boxes + 12, d_boxes);
	if (d.rots) k_local_rotations<<<(d.n_tets + 63) / 64, 64, 0, s>>>(d_verts, d.orig_verts, d.tets, d.n_tets, r.rots.get());
	// 3. TetMesh::build_tet_grid: mark, scan, scatter, order
	uint32_t* d_counts = r.d_counts.get();
	unsigned int* d_n_marks = r.d_n_marks.get();
	unsigned int n_marks = 0;
	for (int attempt = 0; attempt < 2; ++attempt) {
		CU(cudaMemsetAsync(d_counts, 0, (size_t)n_cells * 4, s));
		CU(cudaMemsetAsync(d_n_marks, 0, 4, s));
		k_tet_mark<<<d.n_tets * CASCADES, 128, 0, s>>>(d_verts, d.tets, d.n_tets, d_counts, r.d_marks.get(), (uint32_t)r.d_marks.capacity(), d_n_marks);
		CU(cudaMemcpyAsync(&n_marks, d_n_marks, 4, cudaMemcpyDeviceToHost, s));
		CU(cudaStreamSynchronize(s));  // one sync per edit: the list length decides the allocation
		t_marked = now();
		if (n_marks <= r.d_marks.capacity()) break;
		if (attempt == 1) return fail(NSB_ERR_CUDA, "nsb_cage_deform: mark buffer overflow after regrow");
		CU(r.d_marks.reserve((size_t)n_marks + n_marks / 4));
	}
	// The list outgrew its array: take a larger one before the scan rewrites the offsets. No DevOp, on the host or on the device, points at
	// a freed array: a failed allocation leaves the operator as it was, and the old list (in `idx` after the swap) lives past the DevOp upload.
	DevBuf<uint32_t> idx;
	if ((uint64_t)n_marks > r.lut_idx.capacity() || !r.lut_idx.get()) {
		CU(idx.reserve((size_t)n_marks + n_marks / 4 + 1));
		std::swap(r.lut_idx, idx);
		d.lut_idx = r.lut_idx.get();
	}
	uint32_t* d_off = r.lut_off.get();
	uint32_t* d_idx = r.lut_idx.get();
	k_scan_block_sums<<<n_scan_blocks, SCAN_THREADS, 0, s>>>(d_counts, n_cells, r.d_block_sums.get());
	k_scan_sums<<<1, SCAN_THREADS, 0, s>>>(r.d_block_sums.get(), n_scan_blocks, r.d_total.get());
	k_scan_apply<<<n_scan_blocks, SCAN_THREADS, 0, s>>>(d_counts, n_cells, r.d_block_sums.get(), r.d_total.get(), d_off);
	if (n_marks) {
		k_tet_fill<<<(n_marks + 255) / 256, 256, 0, s>>>(r.d_marks.get(), n_marks, d_off, d_counts, d_idx);
		// the counts are all zero again and the marks are consumed: reuse them as the long-cell queue and the sort scratch
		CU(cudaMemsetAsync(d_n_marks, 0, 4, s));
		k_tet_sort<<<(n_cells + 255) / 256, 256, 0, s>>>(d_off, n_cells, d_idx, d_counts, d_n_marks);
		k_tet_sort_long<<<c->sm_count * 4, 256, 0, s>>>(d_off, d_idx, d_counts, d_n_marks, reinterpret_cast<uint32_t*>(r.d_marks.get()));
	}
	r.n_idx = n_marks;
	// 4. the operator's boxes and (possibly) its list pointer
	float boxes[12];
	t_launched = now();
	CU(cudaMemcpyAsync(boxes, d_boxes, sizeof(boxes), cudaMemcpyDeviceToHost, s));
	CU(cudaStreamSynchronize(s));
	if (verbose)
		fprintf(stderr, "[nsb] cage_deform op %d: %u marks; mark phase %.3f ms, launches %.3f ms, drain %.3f ms\n", op_index, n_marks, t_marked - t_start,
		        t_launched - t_marked, now() - t_launched);
	cp3(d.bmin, boxes); cp3(d.bmax, boxes + 3); cp3(d.wbmin, boxes + 6); cp3(d.wbmax, boxes + 9);
	CU(cudaMemcpyAsync(c->d_ops.get() + op_index, &d, sizeof(DevOp), cudaMemcpyHostToDevice, s));
	CU(cudaGetLastError());
	return NSB_OK;
}
// TetMesh::vanish (tet_mesh.cu:251-363): the cells the operator's current (deformed) tets touch leave the context's running density grid and
// occupancy bitfield, on the stream, with nothing allocated and nothing synchronised unless the count is asked for
extern "C" NsbStatus nsb_cage_vanish(NsbContext* c, int32_t op_index, uint64_t* n_cells_cleared, void* stream_) {
	using namespace nsb::rebuild;
	NsbStatus st = cage_slot(c, op_index, "nsb_cage_vanish");
	if (st != NSB_OK) return st;
	if (!c->has_occ || !c->d_bitfield.get()) return fail(NSB_ERR_STATE, "nsb_cage_vanish: no occupancy (nsb_upload_occupancy, nsb_upload_density_grid or nsb_update_density_grid)");
	CU(cudaSetDevice(c->device));
	cudaStream_t s = (cudaStream_t)stream_;
	const DevOp& d = c->h_ops[op_index];
	float* grid = c->d_density_grid.get();
	uint32_t* bits = reinterpret_cast<uint32_t*>(c->d_bitfield.get());
	const uint32_t n_ctas = d.n_tets * CASCADES;
	if (!n_cells_cleared) {
		k_tet_vanish<<<n_ctas, 128, 0, s>>>(d.verts, d.tets, d.n_tets, grid, bits, 0, nullptr);
		CU(cudaGetLastError());
		return NSB_OK;
	}
	unsigned long long* d_n = c->d_n_cleared.get();
	CU(cudaMemsetAsync(d_n, 0, sizeof(*d_n), s));
	if (grid) k_tet_vanish<<<n_ctas, 128, 0, s>>>(d.verts, d.tets, d.n_tets, grid, bits, 1, nullptr);
	k_tet_vanish<<<n_ctas, 128, 0, s>>>(d.verts, d.tets, d.n_tets, nullptr, bits, 0, d_n);
	unsigned long long n = 0;
	CU(cudaMemcpyAsync(&n, d_n, sizeof(n), cudaMemcpyDeviceToHost, s));
	CU(cudaStreamSynchronize(s));
	*n_cells_cleared = n;
	return NSB_OK;
}
// ---- membrane boundary values (SURVEY.md §8f-4) ---------------------------------------------------------------------
// Host part of GrowingSelection::compute_poisson_boundary (growing_selection.cu:2235-2260): stratified directions on the sphere,
// jittered by a seeded pcg32 instead of the reference's unseeded std::rand(). libm calls as the reference makes them.
static void boundary_coords(const float* points, uint32_t n_points, const NsbBoundarySampling* p, std::vector<float>& coords) {
	const uint32_t w = p->sampling_width, n_sh = w * w;
	coords.assign((size_t)n_points * n_sh * 7, 0.0f);
	Pcg32 rng;
	rng.state = 0u; rng.inc = (0xda3e39cb94b95bdbULL << 1u) | 1u;  // pcg32(seed): tcnn default stream
	rng.next_uint(); rng.state += p->seed; rng.next_uint();
	auto next_float = [&rng] { uint32_t u = (rng.next_uint() >> 9) | 0x3f800000u; float f; memcpy(&f, &u, 4); return f - 1.0f; };
	for (uint32_t k = 0; k < n_points; ++k)
		for (uint32_t i = 0; i < w; ++i)
			for (uint32_t j = 0; j < w; ++j) {
				const float u = ((float)i + next_float()) / (float)p->hemisphere_width;
				const float v = ((float)j + next_float()) / (float)p->hemisphere_width;
				const float theta = (float)(2.f * M_PI * v);
				const float phi = acosf(2.f * u - 1.f);
				const float x = cosf(theta) * sinf(phi), y = sinf(theta) * sinf(phi), z = cosf(phi);
				float* c = coords.data() + ((size_t)n_sh * k + (size_t)i * w + j) * 7;
				for (int a = 0; a < 3; ++a) c[a] = (points[3 * k + a] - p->train_aabb_min[a]) / (p->train_aabb_max[a] - p->train_aabb_min[a]);  // warp_position
				c[4] = (x + 1.0f) * 0.5f; c[5] = (y + 1.0f) * 0.5f; c[6] = (z + 1.0f) * 0.5f;                                                   // warp_direction
			}
}
extern "C" NsbStatus nsb_poisson_boundary(NsbContext* c, const float* points, uint32_t n_points, const NsbBoundarySampling* p, float* density_out, float* shs_out) {
	if (!c || !points || !p || !density_out || !shs_out) return fail(NSB_ERR_INVALID, "nsb_poisson_boundary: null argument");
	if (!c->has_model) return fail(NSB_ERR_STATE, "nsb_upload_model has not been called");
	if (p->sampling_width == 0 || p->sampling_width > 64 || p->hemisphere_width == 0) return fail(NSB_ERR_INVALID, "nsb_poisson_boundary: bad sampling widths");
	if (p->is_inside && !c->has_occ) return fail(NSB_ERR_STATE, "nsb_poisson_boundary: is_inside needs an occupancy grid");
	if (n_points == 0) return NSB_OK;
	CU(cudaSetDevice(c->device));
	const uint32_t n_sh = p->sampling_width * p->sampling_width;
	const uint64_t n64 = (uint64_t)n_points * n_sh;
	if (n64 > 0x7fffff00ull) return fail(NSB_ERR_INVALID, "nsb_poisson_boundary: too many samples");
	const uint32_t n = (uint32_t)n64, n_padded = next_multiple_u32(n, 128u);  // tcnn::batch_size_granularity (:2231)
	std::vector<float> coords;
	boundary_coords(points, n_points, p, coords);
	DevBuf<float> d_coords, d_aabb, d_dens, d_shs;
	DevBuf<__half> d_net;
	CU(d_coords.reserve((size_t)n * 7));
	CU(d_aabb.reserve(6));
	CU(d_dens.reserve(n_points));
	CU(d_shs.reserve((size_t)n_points * 27));
	CU(d_net.reserve((size_t)16 * n_padded));
	CU(cudaMemcpy(d_coords.get(), coords.data(), (size_t)n * 7 * 4, cudaMemcpyHostToDevice));
	float aabb[6] = {p->train_aabb_min[0], p->train_aabb_min[1], p->train_aabb_min[2], p->train_aabb_max[0], p->train_aabb_max[1], p->train_aabb_max[2]};
	CU(cudaMemcpy(d_aabb.get(), aabb, sizeof(aabb), cudaMemcpyHostToDevice));
	(c->acc16 ? k_inference<false, true> : k_inference<false, false>)<<<tile_ctas(c, n_padded, c->inference_ctas_per_sm), 128, sizeof(tc::TileSmem)>>>(c->model, d_coords.get(), n, d_net.get(), n_padded);  // inference_mixed_precision (:2286)
	const float scale = (float)(4 * M_PI / (double)n_sh);                                                // :2341
	nsb::rebuild::k_boundary_fit<<<n_points, 32>>>(d_net.get(), n_padded, d_coords.get(), n_sh, p->rgb_activation, p->density_activation,
	                                               p->is_inside ? c->d_bitfield.get() : nullptr, d_aabb.get(), scale, d_dens.get(), d_shs.get());
	CU(cudaGetLastError());
	CU(cudaMemcpy(density_out, d_dens.get(), (size_t)n_points * 4, cudaMemcpyDeviceToHost));
	CU(cudaMemcpy(shs_out, d_shs.get(), (size_t)n_points * 27 * 4, cudaMemcpyDeviceToHost));
	return NSB_OK;
}
extern "C" NsbStatus nsb_cage_set_membrane(NsbContext* c, int32_t op_index, const float* gamma, uint32_t n_cv, const float* inside_density,
                                           const float* outside_density, const float* inside_shs, const float* outside_shs, float residual_amplitude,
                                           int32_t apply_poisson, float* b_shs_out, float* b_od_out, float* b_rd_out) {
	NsbStatus st = cage_slot(c, op_index, "nsb_cage_set_membrane");
	if (st != NSB_OK) return st;
	if (!gamma || !inside_density || !outside_density || !inside_shs || !outside_shs || n_cv == 0) return fail(NSB_ERR_INVALID, "nsb_cage_set_membrane: null argument");
	CU(cudaSetDevice(c->device));
	CU(cudaDeviceSynchronize());
	DevOp& d = c->h_ops[op_index];
	const uint32_t nv = c->rb[op_index].n_vertices;
	// per-cage-vertex weights on the host, with libm like the reference (:2374-2381)
	std::vector<float> alpha_out(n_cv), w_in(n_cv);
	const float min_step = 1.73205080757f / 1024.0f;  // MIN_CONE_STEPSIZE
	for (uint32_t j = 0; j < n_cv; ++j) {
		const float a_out = 1 - expf(-outside_density[j] * min_step), a_in = 1 - expf(-inside_density[j] * min_step);
		const float q = a_in / a_out;
		alpha_out[j] = a_out;
		w_in[j] = (1.f < q) ? 1.f : q;  // std::min(alpha_in / alpha_out, 1.f)
	}
	const size_t small = (size_t)n_cv * (4 + 54);
	std::vector<float> pack(small);
	memcpy(pack.data(), alpha_out.data(), n_cv * 4);
	memcpy(pack.data() + n_cv, w_in.data(), n_cv * 4);
	memcpy(pack.data() + 2 * (size_t)n_cv, inside_density, n_cv * 4);
	memcpy(pack.data() + 3 * (size_t)n_cv, outside_density, n_cv * 4);
	memcpy(pack.data() + 4 * (size_t)n_cv, inside_shs, (size_t)n_cv * 27 * 4);
	memcpy(pack.data() + 31 * (size_t)n_cv, outside_shs, (size_t)n_cv * 27 * 4);
	auto& r = c->rb[op_index];
	// scratch of the blend, kept with the operator (a host re-blends after every boundary re-sampling) and sized to its cage
	if (r.d_mem_small.capacity() != small) { r.d_gamma = {}; r.d_mem_small = {}; }
	CU(r.d_gamma.reserve((size_t)nv * n_cv));
	CU(r.d_mem_small.reserve(small));
	float* d_small = r.d_mem_small.get();
	CU(cudaMemcpy(r.d_gamma.get(), gamma, (size_t)nv * n_cv * 4, cudaMemcpyHostToDevice));
	CU(cudaMemcpy(d_small, pack.data(), small * 4, cudaMemcpyHostToDevice));
	// the boundary arrays, unless nsb_set_edit_ops uploaded them
	CU(r.shs.reserve((size_t)nv * 27));
	CU(r.od.reserve(nv));
	CU(r.rd.reserve(nv));
	d.shs = r.shs.get(); d.od = r.od.get(); d.rd = r.rd.get();
	dim3 block(32, 4);
	nsb::rebuild::k_membrane_blend<<<(nv + 3) / 4, block>>>(r.d_gamma.get(), nv, n_cv, d_small, d_small + n_cv, d_small + 2 * (size_t)n_cv, d_small + 3 * (size_t)n_cv,
	                                                        d_small + 4 * (size_t)n_cv, d_small + 31 * (size_t)n_cv, r.shs.get(), r.od.get(), r.rd.get());
	CU(cudaGetLastError());
	d.has_poisson_data = 1;
	d.apply_poisson = apply_poisson ? 1 : 0;
	d.amp = residual_amplitude;
	CU(cudaMemcpy(c->d_ops.get() + op_index, &d, sizeof(DevOp), cudaMemcpyHostToDevice));
	int any = 0;
	for (const DevOp& o : c->h_ops) if (o.type == NSB_OP_CAGE && o.apply_poisson && o.has_poisson_data && o.n_tets) any = 1;
	c->any_poisson = any;
	if (b_shs_out) CU(cudaMemcpy(b_shs_out, d.shs, (size_t)nv * 27 * 4, cudaMemcpyDeviceToHost));
	if (b_od_out) CU(cudaMemcpy(b_od_out, d.od, (size_t)nv * 4, cudaMemcpyDeviceToHost));
	if (b_rd_out) CU(cudaMemcpy(b_rd_out, d.rd, (size_t)nv * 4, cudaMemcpyDeviceToHost));
	return NSB_OK;
}
extern "C" NsbStatus nsb_cage_download(NsbContext* c, int32_t op_index, float* vertices, float* rotations, uint32_t* lut_offsets, uint32_t* lut_idx,
                                       uint64_t idx_capacity, uint64_t* n_idx, float* boxes) {
	NsbStatus st = cage_slot(c, op_index, "nsb_cage_download");
	if (st != NSB_OK) return st;
	CU(cudaSetDevice(c->device));
	CU(cudaDeviceSynchronize());
	const DevOp& d = c->h_ops[op_index];
	const auto& r = c->rb[op_index];
	if (vertices) CU(cudaMemcpy(vertices, d.verts, (size_t)3 * r.n_vertices * 4, cudaMemcpyDeviceToHost));
	if (rotations) {
		if (!d.rots) return fail(NSB_ERR_STATE, "nsb_cage_download: operator %d has no local rotations", op_index);
		CU(cudaMemcpy(rotations, d.rots, (size_t)9 * d.n_tets * 4, cudaMemcpyDeviceToHost));
	}
	if (lut_offsets) CU(cudaMemcpy(lut_offsets, d.lut_off, ((size_t)NSB_GRID_CELLS + 1) * 4, cudaMemcpyDeviceToHost));
	if (n_idx) *n_idx = r.n_idx;
	if (lut_idx) {
		if (idx_capacity < r.n_idx) return fail(NSB_ERR_INVALID, "nsb_cage_download: idx buffer too small (%llu needed)", (unsigned long long)r.n_idx);
		if (r.n_idx) CU(cudaMemcpy(lut_idx, d.lut_idx, (size_t)r.n_idx * 4, cudaMemcpyDeviceToHost));
	}
	if (boxes) { cp3(boxes, d.bmin); cp3(boxes + 3, d.bmax); cp3(boxes + 6, d.wbmin); cp3(boxes + 9, d.wbmax); }
	return NSB_OK;
}

// ---- frame conversion ---------------------------------------------------------------------------------
static const uint32_t kSobolDir1[32] = {
	0x80000000, 0xc0000000, 0xa0000000, 0xf0000000, 0x88000000, 0xcc000000, 0xaa000000, 0xff000000, 0x80800000, 0xc0c00000, 0xa0a00000,
	0xf0f00000, 0x88880000, 0xcccc0000, 0xaaaa0000, 0xffff0000, 0x80008000, 0xc000c000, 0xa000a000, 0xf000f000, 0x88008800, 0xcc00cc00,
	0xaa00aa00, 0xff00ff00, 0x80808080, 0xc0c0c0c0, 0xa0a0a0a0, 0xf0f0f0f0, 0x88888888, 0xcccccccc, 0xaaaaaaaa, 0xffffffff,
};
// ld_random_val_2d (random_val.cuh:278-282)
static void host_ld_random_val_2d(uint32_t index, uint32_t seed, float* out) {
	index = nested_uniform_scramble_base2(index, seed);
	for (uint32_t dim = 0; dim < 2; ++dim) {
		uint32_t X = 0;
		for (uint32_t bit = 0; bit < 32; ++bit) {
			uint32_t mask = (index >> bit) & 1u;
			X ^= mask * (dim == 0 ? (0x80000000u >> bit) : kSobolDir1[bit]);
		}
		out[dim] = (float)nested_uniform_scramble_base2(X, hash_combine(seed, dim)) * 2.3283064365386963e-10f;
	}
}
// ld_random_pixel_offset (random_val.cuh:317-322): the same for every pixel, so evaluated once here
static void host_pixel_offset(uint32_t spp, float* off) {
	float a[2], b[2];
	host_ld_random_val_2d(0, 0xdeadbeefu, a);
	host_ld_random_val_2d(spp, 0xdeadbeefu, b);
	for (int i = 0; i < 2; ++i) {
		volatile float s = 0.5f - a[i];
		volatile float o = s + b[i];
		off[i] = o - floorf(o);
	}
}

static NsbStatus to_dev_frame(const NsbFrame* f, DevFrame* d) {
	if (!f) return fail(NSB_ERR_INVALID, "frame is null");
	if (f->width <= 0 || f->height <= 0 || (uint64_t)f->width * f->height > 0x7fffffffull / 786433ull * 786433ull) return fail(NSB_ERR_INVALID, "bad resolution %dx%d", f->width, f->height);
	if (f->tile_world <= 0 || f->tile_rank < 0 || f->tile_rank >= f->tile_world) return fail(NSB_ERR_INVALID, "bad tile partition %d/%d", f->tile_rank, f->tile_world);
	switch (f->render_mode) {
		case NSB_RENDER_AO: case NSB_RENDER_SHADE: case NSB_RENDER_POSITIONS: case NSB_RENDER_DEPTH:
		case NSB_RENDER_DISTANCE: case NSB_RENDER_STEPSIZE: case NSB_RENDER_COST: case NSB_RENDER_DISTORTION: break;
		default: return fail(NSB_ERR_UNSUPPORTED, "render mode %d is not covered (Normals/EncodingVis need network input gradients; Slice is a side path)", f->render_mode);
	}
	if (f->camera_distortion_mode < 0 || f->camera_distortion_mode > 2) return fail(NSB_ERR_INVALID, "bad camera distortion mode %d", f->camera_distortion_mode);
	if (f->focus_z < 0.0f) return fail(NSB_ERR_UNSUPPORTED, "negative focus_z selects the reference's Slice side path (testbed_nerf.cu:3067-3070), which is not covered");
	if (f->dof != 0.0f && !(f->focus_z > 0.0f)) return fail(NSB_ERR_INVALID, "depth of field needs focus_z > 0");
	if (f->envmap_dev && (f->envmap_resolution[0] <= 0 || f->envmap_resolution[1] <= 0)) return fail(NSB_ERR_INVALID, "bad envmap resolution");
	if (f->distortion_dev && (f->distortion_resolution[0] <= 0 || f->distortion_resolution[1] <= 0)) return fail(NSB_ERR_INVALID, "bad distortion map resolution");
	if (f->rgb_activation < 0 || f->rgb_activation > 3 || f->density_activation < 0 || f->density_activation > 3) return fail(NSB_ERR_INVALID, "bad activation");
	d->W = f->width; d->H = f->height;
	d->fx = f->focal_length[0]; d->fy = f->focal_length[1];
	d->cx = f->screen_center[0]; d->cy = f->screen_center[1];
	memcpy(d->cam0, f->camera0, sizeof(d->cam0));
	memcpy(d->cam1, f->camera1, sizeof(d->cam1));
	memcpy(d->rs, f->rolling_shutter, sizeof(d->rs));
	cp3(d->rmin, f->render_aabb_min); cp3(d->rmax, f->render_aabb_max);
	cp3(d->tmin, f->train_aabb_min); cp3(d->tmax, f->train_aabb_max);
	d->tinv_exact = 1;
	for (int a = 0; a < 3; ++a) {  // the extent as the device computes it (one fp32 subtraction); 2^k with a normal 2^-k: store 2^-k
		const float e = d->tmax[a] - d->tmin[a];
		uint32_t b;
		memcpy(&b, &e, sizeof(b));
		const uint32_t ex = b >> 23;  // sign and exponent field: e > 0 has no sign bit
		const bool pow2 = (b & 0x7fffffu) == 0 && ex >= 1 && ex <= 253;
		const uint32_t ib = (254u - ex) << 23;
		if (pow2) memcpy(&d->tinv[a], &ib, sizeof(ib));
		else d->tinv[a] = 0.0f;
		d->tinv_exact &= pow2 ? 1 : 0;
	}
	d->cone = f->cone_angle_constant;
	d->min_T = f->min_transmittance;
	d->depth_scale = f->depth_scale;
	d->rgb_act = f->rgb_activation; d->density_act = f->density_activation; d->mode = f->render_mode;
	d->spp = f->spp_index;
	host_pixel_offset(f->snap_to_pixel_centers ? 0u : f->spp_index, d->pix_off);
	d->apply_ops = f->apply_operators; d->poisson_target = f->poisson_target; d->linear_colors = f->linear_colors;
	d->min_mip = f->min_mip < 0 ? 0 : (f->min_mip > 4 ? 4 : f->min_mip);
	d->show_accel = f->show_accel != 0;
	d->tile_rank = f->tile_rank; d->tile_world = f->tile_world;
	d->tiles_x = (f->width + TILE_W - 1) / TILE_W;
	d->tiles_y = (f->height + TILE_H - 1) / TILE_H;
	d->cam_dist_mode = f->camera_distortion_mode;
	memcpy(d->cam_dist, f->camera_distortion_params, sizeof(d->cam_dist));
	d->dof = f->dof; d->focus_z = f->focus_z;
	d->glow_mode = f->glow_mode; d->glow_y_cutoff = f->glow_y_cutoff;
	d->envmap = f->envmap_dev; d->env_w = f->envmap_resolution[0]; d->env_h = f->envmap_resolution[1];
	d->distortion = f->distortion_dev; d->dist_w = f->distortion_resolution[0]; d->dist_h = f->distortion_resolution[1];
	d->general_camera = (d->cam_dist_mode != 0 || d->distortion != nullptr || d->dof != 0.0f) ? 1 : 0;
	return NSB_OK;
}

// The frame's render AABB lies inside its train AABB (a NaN bound fails the test).
static bool render_in_range(const DevFrame& f) {
	for (int a = 0; a < 3; ++a)
		if (!(f.rmin[a] >= f.tmin[a] && f.rmax[a] <= f.tmax[a])) return false;
	return true;
}

extern "C" NsbStatus nsb_render(NsbContext* c, const NsbFrame* frame, float* fb_dev, float* depth_dev, void* stream_) {
	if (!c || !fb_dev || !depth_dev) return fail(NSB_ERR_INVALID, "null argument");
	if (!c->has_model) return fail(NSB_ERR_STATE, "nsb_upload_model has not been called");
	DevFrame f;
	NsbStatus st = to_dev_frame(frame, &f);
	if (st != NSB_OK) return st;
	CU(cudaSetDevice(c->device));
	cudaStream_t stream = (cudaStream_t)stream_;
	uint32_t n_tiles = (uint32_t)(f.tiles_x * f.tiles_y);
	uint32_t my_tiles = (n_tiles + (uint32_t)f.tile_world - 1 - (uint32_t)f.tile_rank) / (uint32_t)f.tile_world;
	size_t n_local = (size_t)my_tiles * TILE_PIXELS;
	if (n_local > c->d_list.capacity()) {
		CU(cudaStreamSynchronize(stream));
		CU(c->d_list.reserve(n_local));
	}
	// frames whose ray generation is not the pinhole fast path (ABI 3): k_prepare_rays<true>; with a general camera the rays travel in a side buffer
	const bool general = f.general_camera || f.envmap != nullptr || f.mode == NSB_RENDER_DISTORTION;
	float* ray_od = nullptr;
	if (f.general_camera) {
		if (n_local * 6 > c->d_ray_od.capacity()) {
			CU(cudaStreamSynchronize(stream));
			CU(c->d_ray_od.reserve(n_local * 6));
		}
		ray_od = c->d_ray_od.get();
	}
	const uint8_t* bitfield = c->has_occ ? c->d_bitfield.get() : nullptr;
	RayRec* list = c->d_list.get();
	uint32_t* counters = c->d_counters.get();
	unsigned long long* stats = c->d_stats.get();
	CU(cudaEventRecord(c->ev0, stream));
	CU(cudaEventRecord(c->evm, stream));
	CU(cudaMemsetAsync(counters, 0, 2 * sizeof(uint32_t), stream));
	CU(cudaMemsetAsync(stats, 0, ST_N * sizeof(unsigned long long), stream));
	if (n_local > 0) {
		if (general)
			k_prepare_rays<true><<<(unsigned)((n_local + 255) / 256), 256, 0, stream>>>(f, bitfield, reinterpret_cast<float4*>(fb_dev), depth_dev, list, ray_od, counters,
			                                                                         (uint32_t)n_local, stats);
		else
			k_prepare_rays<false><<<(unsigned)((n_local + 255) / 256), 256, 0, stream>>>(f, bitfield, reinterpret_cast<float4*>(fb_dev), depth_dev, list, nullptr, counters,
			                                                                          (uint32_t)n_local, stats);
		CU(cudaGetLastError());
		CU(cudaEventRecord(c->evm, stream));
		const bool ops_on = f.apply_ops && c->n_ops > 0;
		const uint32_t tiles = (uint32_t)render_tiles(ops_on, c->acc16);
		uint32_t grid = (uint32_t)c->sm_count;  // one CTA per SM
		if (grid > (my_tiles + tiles - 1) / tiles) grid = (my_tiles + tiles - 1) / tiles;
		// The in-range grid index (nsb_device.cuh) is exact for this frame when render_in_range holds. Without operators the fused kernel
		// encodes only march samples, and the march hands out only positions inside the render AABB (box_contains). With the render AABB
		// inside the train AABB, warp_position and warp_position_pow2 (both monotone) map every such position into [0, 1] up to rounding,
		// well inside [-0.5/scale, 1 + 0.5/scale]. So every grid coordinate is at most res, and dense_in_range bounds the dense index by 2*size.
		const bool in_range = !ops_on && c->dense_in_range && render_in_range(f);
		auto kernel = ops_on ? (c->acc16 ? k_render_fused<true, true, false> : k_render_fused<true, false, false>)
		                     : in_range ? (c->acc16 ? k_render_fused<false, true, true> : k_render_fused<false, false, true>)
		                                : (c->acc16 ? k_render_fused<false, true, false> : k_render_fused<false, false, false>);
		const size_t smem = ops_on ? sizeof(RenderSmemT<render_tiles(true, false)>)
		                           : c->acc16 ? sizeof(RenderSmemT<render_tiles(false, true)>) : sizeof(RenderSmemT<render_tiles(false, false)>);
		kernel<<<grid, 128 * tiles, smem, stream>>>(f, c->model, bitfield, c->d_ops.get(), c->n_ops, c->any_poisson,
		                                                          reinterpret_cast<float4*>(fb_dev), depth_dev, list, ray_od, counters, counters + 1, stats);
		CU(cudaGetLastError());
	}
	CU(cudaEventRecord(c->ev1, stream));
	c->timed = true;
	c->launches = 2;
	return NSB_OK;
}

extern "C" NsbStatus nsb_render_host(NsbContext* c, const NsbFrame* frame, float* fb_host, float* depth_host) {
	if (!c || !frame || !fb_host) return fail(NSB_ERR_INVALID, "null argument");
	CU(cudaSetDevice(c->device));
	size_t n = (size_t)frame->width * (size_t)frame->height;
	if (n == 0) return fail(NSB_ERR_INVALID, "empty frame");
	CU(c->d_fb.reserve(n * 4));
	CU(c->d_depth.reserve(n));
	float* fb = c->d_fb.get();
	float* depth = c->d_depth.get();
	CU(cudaMemsetAsync(fb, 0, n * 16, c->stream));  // render_buffer.clear_frame (testbed.cu:2635)
	CU(cudaMemsetAsync(depth, 0, n * 4, c->stream));
	NsbStatus st = nsb_render(c, frame, fb, depth, c->stream);
	if (st != NSB_OK) return st;
	CU(cudaMemcpyAsync(fb_host, fb, n * 16, cudaMemcpyDeviceToHost, c->stream));
	if (depth_host) CU(cudaMemcpyAsync(depth_host, depth, n * 4, cudaMemcpyDeviceToHost, c->stream));
	CU(cudaStreamSynchronize(c->stream));
	return NSB_OK;
}

extern "C" NsbStatus nsb_render_host_async(NsbContext* c, const NsbFrame* frame, float* fb_host, float* depth_host, uint64_t* ticket) {
	if (!c || !frame || !fb_host || !ticket) return fail(NSB_ERR_INVALID, "null argument");
	CU(cudaSetDevice(c->device));
	const size_t n = (size_t)frame->width * (size_t)frame->height;
	if (n == 0) return fail(NSB_ERR_INVALID, "empty frame");
	if (c->d_fb2[0].capacity() < n * 4 || c->d_fb2[1].capacity() < n * 4 || c->d_depth2[0].capacity() < n || c->d_depth2[1].capacity() < n) {
		CU(cudaStreamSynchronize(c->stream));
		CU(cudaStreamSynchronize(c->copy_stream));
		for (int i = 0; i < 2; ++i) {
			CU(c->d_fb2[i].reserve(n * 4));
			CU(c->d_depth2[i].reserve(n));
		}
	}
	const int slot = (int)(c->host_seq & 1u);
	float* fb = c->d_fb2[slot].get();
	float* depth = c->d_depth2[slot].get();
	if (c->host_seq >= 2) CU(cudaStreamWaitEvent(c->stream, c->copy_done[slot], 0));  // the copy that last read this slot (two tickets ago)
	CU(cudaMemsetAsync(fb, 0, n * 16, c->stream));  // render_buffer.clear_frame (testbed.cu:2635)
	CU(cudaMemsetAsync(depth, 0, n * 4, c->stream));
	NsbStatus st = nsb_render(c, frame, fb, depth, c->stream);
	if (st != NSB_OK) return st;
	CU(cudaEventRecord(c->render_done[slot], c->stream));
	CU(cudaStreamWaitEvent(c->copy_stream, c->render_done[slot], 0));
	CU(cudaMemcpyAsync(fb_host, fb, n * 16, cudaMemcpyDeviceToHost, c->copy_stream));
	if (depth_host) CU(cudaMemcpyAsync(depth_host, depth, n * 4, cudaMemcpyDeviceToHost, c->copy_stream));
	CU(cudaEventRecord(c->copy_done[slot], c->copy_stream));
	*ticket = c->host_seq++;
	return NSB_OK;
}

extern "C" NsbStatus nsb_host_frame_wait(NsbContext* c, uint64_t ticket) {
	if (!c) return fail(NSB_ERR_INVALID, "null context");
	if (ticket >= c->host_seq) return fail(NSB_ERR_INVALID, "ticket %llu was never issued", (unsigned long long)ticket);
	CU(cudaSetDevice(c->device));
	CU(cudaEventSynchronize(c->copy_done[ticket & 1u]));  // if the slot was reused since, this is the later copy, which started after this one finished
	return NSB_OK;
}

extern "C" NsbStatus nsb_set_mlp_accumulator(NsbContext* c, int32_t policy) {
	if (!c) return fail(NSB_ERR_INVALID, "null context");
	if (policy != NSB_MLP_ACC_F32 && policy != NSB_MLP_ACC_F16) return fail(NSB_ERR_INVALID, "unknown accumulator policy %d", policy);
	c->acc16 = policy == NSB_MLP_ACC_F16;
	return NSB_OK;
}

extern "C" NsbStatus nsb_get_stats(NsbContext* c, NsbRenderStats* out) {
	if (!c || !out) return fail(NSB_ERR_INVALID, "null argument");
	CU(cudaSetDevice(c->device));
	memset(out, 0, sizeof(*out));
	if (!c->timed) return NSB_OK;
	CU(cudaEventSynchronize(c->ev1));
	unsigned long long h[ST_N];
	CU(cudaMemcpy(h, c->d_stats.get(), sizeof(h), cudaMemcpyDeviceToHost));
	out->n_rays = h[ST_RAYS]; out->n_rays_alive = h[ST_ALIVE]; out->n_hit = h[ST_HIT]; out->n_samples = h[ST_SAMPLES]; out->n_old_samples = h[ST_OLD];
	out->n_kernel_launches = c->launches;
	CU(cudaEventElapsedTime(&out->gpu_ms, c->ev0, c->ev1));
	CU(cudaEventElapsedTime(&out->fused_ms, c->evm, c->ev1));
	return NSB_OK;
}

// Diagnostic counters of the last render, per render tile (thread 0 of each 128-thread tile adds them): rounds (tile x MLP rounds),
// and cycles per phase summed over tiles: {rounds, acquire, encode, mlp, composite, total, tiles}
extern "C" NsbStatus nsb_debug_counters(NsbContext* c, uint64_t* out, int32_t n) {
	if (!c || !out || n < 7) return fail(NSB_ERR_INVALID, "need room for 7 counters");
	CU(cudaSetDevice(c->device));
	if (c->timed) CU(cudaEventSynchronize(c->ev1));
	unsigned long long h[ST_N];
	CU(cudaMemcpy(h, c->d_stats.get(), sizeof(h), cudaMemcpyDeviceToHost));
	for (int i = 0; i < 7; ++i) out[i] = h[ST_ROUNDS + i];
	return NSB_OK;
}

extern "C" NsbStatus nsb_tiles_for_rank(int32_t width, int32_t height, int32_t rank, int32_t world, uint32_t* n_tiles) {
	if (!n_tiles || width <= 0 || height <= 0 || world <= 0 || rank < 0 || rank >= world) return fail(NSB_ERR_INVALID, "bad arguments");
	uint32_t total = (uint32_t)(((width + TILE_W - 1) / TILE_W) * ((height + TILE_H - 1) / TILE_H));
	*n_tiles = (total + (uint32_t)world - 1 - (uint32_t)rank) / (uint32_t)world;
	return NSB_OK;
}

static NsbStatus pack_impl(NsbContext* c, const float* fb, const float* depth, int W, int H, int rank, int world, float* pr, float* pd, void* stream, int unpack) {
	if (!c || !fb || !pr) return fail(NSB_ERR_INVALID, "null argument");
	uint32_t mine = 0;
	NsbStatus st = nsb_tiles_for_rank(W, H, rank, world, &mine);
	if (st != NSB_OK) return st;
	CU(cudaSetDevice(c->device));
	int tiles_x = (W + TILE_W - 1) / TILE_W, tiles_y = (H + TILE_H - 1) / TILE_H;
	if (mine == 0) return NSB_OK;
	k_pack_tiles<<<mine, TILE_PIXELS, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(fb), depth, W, H, tiles_x, tiles_x * tiles_y, rank, world,
	                                                            reinterpret_cast<float4*>(pr), pd, unpack);
	CU(cudaGetLastError());
	return NSB_OK;
}
extern "C" NsbStatus nsb_pack_tiles(NsbContext* c, const float* fb_dev, const float* depth_dev, int32_t W, int32_t H, int32_t rank, int32_t world,
                                    float* dst_rgba, float* dst_depth, void* stream) {
	return pack_impl(c, fb_dev, depth_dev, W, H, rank, world, dst_rgba, dst_depth, stream, 0);
}
extern "C" NsbStatus nsb_unpack_tiles(NsbContext* c, const float* src_rgba, const float* src_depth, int32_t W, int32_t H, int32_t rank, int32_t world,
                                      float* fb_dev, float* depth_dev, void* stream) {
	return pack_impl(c, fb_dev, depth_dev, W, H, rank, world, const_cast<float*>(src_rgba), const_cast<float*>(src_depth), stream, 1);
}

extern "C" NsbStatus nsb_unpack_gathered(NsbContext* c, const float* gathered_rgba, const float* gathered_depth, int32_t W, int32_t H, int32_t skip_rank, int32_t world,
                                         uint32_t rank_stride_floats, float* fb_dev, float* depth_dev, void* stream) {
	if (!c || !gathered_rgba || !fb_dev || W <= 0 || H <= 0 || world <= 0) return fail(NSB_ERR_INVALID, "bad arguments");
	CU(cudaSetDevice(c->device));
	const int tiles_x = (W + TILE_W - 1) / TILE_W, tiles_y = (H + TILE_H - 1) / TILE_H;
	const uint32_t need = (uint32_t)((tiles_x * tiles_y + world - 1) / world);
	if (rank_stride_floats % 4 != 0 || rank_stride_floats < need * (uint32_t)TILE_PIXELS * 4u) return fail(NSB_ERR_INVALID, "rank stride %u floats is not a multiple of 4 or smaller than rank 0's %u tiles", rank_stride_floats, need);
	k_unpack_gathered<<<dim3(need, (unsigned)world), TILE_PIXELS, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(gathered_rgba), gathered_depth, W, H, tiles_x, tiles_x * tiles_y,
	                                                                                         skip_rank, world, rank_stride_floats, reinterpret_cast<float4*>(fb_dev), depth_dev);
	CU(cudaGetLastError());
	return NSB_OK;
}

extern "C" NsbStatus nsb_accumulate(NsbContext* c, const float* frame, float* acc, int32_t W, int32_t H, uint32_t spp, int32_t color_space, void* stream) {
	if (!c || !frame || !acc || W <= 0 || H <= 0) return fail(NSB_ERR_INVALID, "bad arguments");
	if (color_space < 0 || color_space > 2) return fail(NSB_ERR_INVALID, "bad colour space %d", color_space);
	CU(cudaSetDevice(c->device));
	int n = W * H;
	if (spp == 0) CU(cudaMemsetAsync(acc, 0, (size_t)n * 16, (cudaStream_t)stream));  // render_buffer.cu:545-547
	k_accumulate<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(n, reinterpret_cast<const float4*>(frame), reinterpret_cast<float4*>(acc), (float)spp, color_space);
	CU(cudaGetLastError());
	return NSB_OK;
}
extern "C" NsbStatus nsb_tonemap(NsbContext* c, const float* acc, float* out, int32_t W, int32_t H, const NsbTonemap* p, void* stream) {
	if (!c || !acc || !out || !p || W <= 0 || H <= 0) return fail(NSB_ERR_INVALID, "bad arguments");
	if (p->color_space < 0 || p->color_space > 2 || p->output_color_space < 0 || p->output_color_space > 1 || p->tonemap_curve < 0 || p->tonemap_curve > 3)
		return fail(NSB_ERR_INVALID, "bad tonemap parameters");
	CU(cudaSetDevice(c->device));
	int n = W * H;
	k_tonemap<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(n, reinterpret_cast<const float4*>(acc), reinterpret_cast<float4*>(out), *p);
	CU(cudaGetLastError());
	return NSB_OK;
}

// ---- whole output frames (ABI 8): Testbed::render_to_cpu's sub-frame loop and run.py's 8-bit conversion ------------------
// the parameter check nsb_tonemap makes inline (kept there unchanged): the two must stay the same
static bool tonemap_ok(const NsbTonemap* p) {
	return p->color_space >= 0 && p->color_space <= 2 && p->output_color_space >= 0 && p->output_color_space <= 1 && p->tonemap_curve >= 0 && p->tonemap_curve <= 3;
}

extern "C" NsbStatus nsb_render_accumulate(NsbContext* c, const NsbFrame* frames, uint32_t n, const NsbTonemap* tm, float* acc, float* out, void* stream_) {
	if (!c || !frames || n == 0 || !tm || !acc || !out) return fail(NSB_ERR_INVALID, "null argument or no sub-frames");
	if (!c->has_model) return fail(NSB_ERR_STATE, "nsb_upload_model has not been called");
	for (uint32_t i = 0; i < n; ++i) {  // every frame as nsb_render checks it, before anything is enqueued
		DevFrame f;
		const NsbStatus st = to_dev_frame(&frames[i], &f);
		if (st != NSB_OK) return fail(st, "nsb_render_accumulate: sub-frame %u: %s", i, g_last_error.c_str());
		if (frames[i].width != frames[0].width || frames[i].height != frames[0].height)
			return fail(NSB_ERR_INVALID, "nsb_render_accumulate: sub-frame %u is %dx%d, sub-frame 0 is %dx%d", i, frames[i].width, frames[i].height, frames[0].width, frames[0].height);
	}
	if (!tonemap_ok(tm)) return fail(NSB_ERR_INVALID, "bad tonemap parameters");
	CU(cudaSetDevice(c->device));
	cudaStream_t stream = (cudaStream_t)stream_;
	const int W = frames[0].width, H = frames[0].height, np = W * H;
	const size_t n_px = (size_t)np;
	if (c->d_sub_fb.capacity() < n_px * 4 || c->d_sub_depth.capacity() < n_px) {  // grows only; the old buffers may still be read on `stream`
		CU(cudaStreamSynchronize(stream));
		CU(c->d_sub_fb.reserve(n_px * 4));
		CU(c->d_sub_depth.reserve(n_px));
	}
	float* fb = c->d_sub_fb.get();
	float* depth = c->d_sub_depth.get();
	for (uint32_t i = 0; i < n; ++i) {  // render_frame (testbed.cu:2632-2765) per sub-frame: clear_frame, render_nerf, accumulate
		CU(cudaMemsetAsync(fb, 0, n_px * 16, stream));
		CU(cudaMemsetAsync(depth, 0, n_px * 4, stream));
		const NsbStatus st = nsb_render(c, &frames[i], fb, depth, stream);
		if (st != NSB_OK) return st;
		const uint32_t spp = frames[i].spp_index;
		if (spp == 0) CU(cudaMemsetAsync(acc, 0, n_px * 16, stream));  // render_buffer.cu:545-547
		k_accumulate<<<(np + 255) / 256, 256, 0, stream>>>(np, reinterpret_cast<const float4*>(fb), reinterpret_cast<float4*>(acc), (float)spp, tm->color_space);
		CU(cudaGetLastError());
	}
	k_tonemap<<<(np + 255) / 256, 256, 0, stream>>>(np, reinterpret_cast<const float4*>(acc), reinterpret_cast<float4*>(out), *tm);
	CU(cudaGetLastError());
	return NSB_OK;
}

extern "C" NsbStatus nsb_frame_to_rgba8(NsbContext* c, const float* rgba, int32_t W, int32_t H, float exposure, int32_t n_channels, uint8_t* out, void* stream) {
	if (!c || !rgba || !out || W <= 0 || H <= 0) return fail(NSB_ERR_INVALID, "bad arguments");
	if ((uint64_t)W * (uint64_t)H > 0xffffffffull) return fail(NSB_ERR_INVALID, "frame %dx%d has more than 2^32 pixels", W, H);
	if (n_channels != 3 && n_channels != 4) return fail(NSB_ERR_INVALID, "n_channels must be 3 or 4, not %d", n_channels);
	if (n_channels == 4 && ((uintptr_t)out & 3u) != 0) return fail(NSB_ERR_INVALID, "a 4-channel output must be 4-byte aligned");
	if (((uintptr_t)rgba & 15u) != 0) return fail(NSB_ERR_INVALID, "the float4 frame must be 16-byte aligned");
	CU(cudaSetDevice(c->device));
	const uint32_t n = (uint32_t)W * (uint32_t)H;
	const float scale = (float)std::pow(2.0, (double)exposure);  // run.py's 2**exposure: a Python float, rounded to float32 against the float32 frame
	video::k_rgba8<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(n, reinterpret_cast<const float4*>(rgba), scale, n_channels, out);
	CU(cudaGetLastError());
	return NSB_OK;
}

// ---- operator-level entry points -------------------------------------------------------------------------
template <bool DENSITY_ONLY>
static NsbStatus inference_impl(NsbContext* c, const float* coords, uint32_t n, uint16_t* out, uint32_t n_padded, void* stream) {
	if (!c) return fail(NSB_ERR_INVALID, "null context");
	if (!c->has_model) return fail(NSB_ERR_STATE, "nsb_upload_model has not been called");
	if (n_padded < n || n_padded % 128 != 0) return fail(NSB_ERR_INVALID, "n_padded must be a multiple of 128 (tcnn::batch_size_granularity) and >= n");
	if (n_padded == 0) return NSB_OK;  // empty batch
	if (!coords || !out) return fail(NSB_ERR_INVALID, "null argument");
	CU(cudaSetDevice(c->device));
	(c->acc16 ? k_inference<DENSITY_ONLY, true> : k_inference<DENSITY_ONLY, false>)<<<tile_ctas(c, n_padded, c->inference_ctas_per_sm), 128, sizeof(tc::TileSmem), (cudaStream_t)stream>>>(c->model, coords, n, reinterpret_cast<__half*>(out), n_padded);
	CU(cudaGetLastError());
	return NSB_OK;
}
extern "C" NsbStatus nsb_inference(NsbContext* c, const float* coords, uint32_t n, uint16_t* out, uint32_t n_padded, void* stream) {
	return inference_impl<false>(c, coords, n, out, n_padded, stream);
}
extern "C" NsbStatus nsb_density(NsbContext* c, const float* coords, uint32_t n, uint16_t* out, uint32_t n_padded, void* stream) {
	return inference_impl<true>(c, coords, n, out, n_padded, stream);
}
extern "C" NsbStatus nsb_encode(NsbContext* c, const float* coords, uint32_t n, uint16_t* out, uint32_t n_padded, void* stream) {
	if (!c || !coords || !out) return fail(NSB_ERR_INVALID, "null argument");
	if (!c->has_model) return fail(NSB_ERR_STATE, "nsb_upload_model has not been called");
	if (n_padded < n) return fail(NSB_ERR_INVALID, "n_padded < n");
	if (n == 0) return NSB_OK;
	CU(cudaSetDevice(c->device));
	k_encode<<<(n + 255) / 256, 256, 0, (cudaStream_t)stream>>>(c->model, coords, n, reinterpret_cast<__half*>(out), n_padded);
	CU(cudaGetLastError());
	return NSB_OK;
}
// op_index < 0: every uploaded operator in reverse list order (the loops of testbed_nerf.cu:2868-2904, outputs cleared first like :2863-2866, :2898);
// op_index >= 0: that operator alone = one EditOperator virtual call (outputs are not cleared, as the virtuals do not clear them)
static NsbStatus op_range(NsbContext* c, int32_t op_index, const DevOp** ops, int* n_ops) {
	if (op_index >= c->n_ops) return fail(NSB_ERR_INVALID, "operator %d of %d", op_index, c->n_ops);
	*ops = op_index < 0 ? c->d_ops.get() : c->d_ops.get() + op_index;
	*n_ops = op_index < 0 ? c->n_ops : 1;
	return NSB_OK;
}
extern "C" NsbStatus nsb_map_rays_op(NsbContext* c, int32_t op_index, float* coords, uint8_t* empty_mask, uint32_t n, void* stream) {
	if (!c || !coords || !empty_mask) return fail(NSB_ERR_INVALID, "null argument");
	if (n == 0) return NSB_OK;
	CU(cudaSetDevice(c->device));
	if (op_index < 0) CU(cudaMemsetAsync(empty_mask, 0, n, (cudaStream_t)stream));  // :2898
	if (c->n_ops == 0) return NSB_OK;
	const DevOp* ops; int n_ops;
	NsbStatus st = op_range(c, op_index, &ops, &n_ops);
	if (st != NSB_OK) return st;
	k_map_rays<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(ops, n_ops, coords, empty_mask, n);
	CU(cudaGetLastError());
	return NSB_OK;
}
extern "C" NsbStatus nsb_map_rays(NsbContext* c, float* coords, uint8_t* empty_mask, uint32_t n, void* stream) { return nsb_map_rays_op(c, -1, coords, empty_mask, n, stream); }
extern "C" NsbStatus nsb_poisson_residuals_op(NsbContext* c, int32_t op_index, const float* coords, uint32_t n, float* sh, float* od, float* rd, void* stream) {
	if (!c || !coords || !sh || !od || !rd) return fail(NSB_ERR_INVALID, "null argument");
	if (n == 0) return NSB_OK;
	CU(cudaSetDevice(c->device));
	if (op_index < 0) {  // :2863-2866
		CU(cudaMemsetAsync(sh, 0, (size_t)n * 27 * sizeof(float), (cudaStream_t)stream));
		CU(cudaMemsetAsync(od, 0, (size_t)n * sizeof(float), (cudaStream_t)stream));
		CU(cudaMemsetAsync(rd, 0, (size_t)n * sizeof(float), (cudaStream_t)stream));
	}
	if (c->n_ops == 0) return NSB_OK;
	const DevOp* ops; int n_ops;
	NsbStatus st = op_range(c, op_index, &ops, &n_ops);
	if (st != NSB_OK) return st;
	k_poisson<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(ops, n_ops, coords, n, sh, od, rd);
	CU(cudaGetLastError());
	return NSB_OK;
}
extern "C" NsbStatus nsb_poisson_residuals(NsbContext* c, const float* coords, uint32_t n, float* sh, float* od, float* rd, void* stream) {
	return nsb_poisson_residuals_op(c, -1, coords, n, sh, od, rd, stream);
}
extern "C" NsbStatus nsb_map_positions(NsbContext* c, int32_t op_index, float* positions, uint32_t stride_floats, uint8_t* empty_mask, uint32_t n, void* stream) {
	if (!c || !positions || stride_floats < 3) return fail(NSB_ERR_INVALID, "bad arguments");
	if (n == 0) return NSB_OK;
	CU(cudaSetDevice(c->device));
	if (op_index < 0 && empty_mask) CU(cudaMemsetAsync(empty_mask, 0, n, (cudaStream_t)stream));  // :3595
	if (c->n_ops == 0) return NSB_OK;
	const DevOp* ops; int n_ops;
	NsbStatus st = op_range(c, op_index, &ops, &n_ops);
	if (st != NSB_OK) return st;
	k_map_positions<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(ops, n_ops, positions, stride_floats, empty_mask, n);
	CU(cudaGetLastError());
	return NSB_OK;
}
extern "C" NsbStatus nsb_poisson_residual_density(NsbContext* c, int32_t op_index, const float* positions, uint32_t stride_floats, uint16_t* density_fp16, uint32_t n, void* stream) {
	if (!c || !positions || !density_fp16 || stride_floats < 3) return fail(NSB_ERR_INVALID, "bad arguments");
	if (n == 0 || c->n_ops == 0) return NSB_OK;
	CU(cudaSetDevice(c->device));
	const DevOp* ops; int n_ops;
	NsbStatus st = op_range(c, op_index, &ops, &n_ops);
	if (st != NSB_OK) return st;
	k_poisson_residual_density<<<(n + 127) / 128, 128, 0, (cudaStream_t)stream>>>(ops, n_ops, positions, stride_floats, reinterpret_cast<__half*>(density_fp16), n);
	CU(cudaGetLastError());
	return NSB_OK;
}
extern "C" NsbStatus nsb_march_trace(NsbContext* c, const NsbFrame* frame, const uint32_t* pixels, uint32_t n_pixels, uint32_t max_samples, float* rec,
                                     uint32_t* idx, uint32_t* count, void* stream) {
	if (!c || !pixels || !rec || !idx || !count) return fail(NSB_ERR_INVALID, "null argument");
	DevFrame f;
	NsbStatus st = to_dev_frame(frame, &f);
	if (st != NSB_OK) return st;
	if (n_pixels == 0) return NSB_OK;
	CU(cudaSetDevice(c->device));
	const uint8_t* bitfield = c->has_occ ? c->d_bitfield.get() : nullptr;
	if (f.general_camera) k_march_trace<true><<<(n_pixels + 63) / 64, 64, 0, (cudaStream_t)stream>>>(f, bitfield, pixels, n_pixels, max_samples, rec, idx, count);
	else k_march_trace<false><<<(n_pixels + 63) / 64, 64, 0, (cudaStream_t)stream>>>(f, bitfield, pixels, n_pixels, max_samples, rec, idx, count);
	CU(cudaGetLastError());
	return NSB_OK;
}

// ---- mesh extraction (Testbed::marching_cubes, testbed_nerf.cu:4614-4649) -------------------------------------------------
static bool grid_res_ok(const int32_t* res) {  // positive multiples of 16 (testbed_nerf.cu:4615-4617) whose point count, padded to 128, fits 32 bits
	for (int a = 0; a < 3; ++a)
		if (res[a] <= 0 || res[a] % 16 != 0) return false;
	return (uint64_t)res[0] * (uint64_t)res[1] * (uint64_t)res[2] <= 0xffffffffull - 127ull;
}

static mesh::GridQuery grid_query(const NsbGridQuery* q) {
	mesh::GridQuery g;
	for (int a = 0; a < 3; ++a) {
		g.res[a] = (uint32_t)q->res[a];
		g.inv_res[a] = 1.0f / (float)q->res[a];
		g.rmin[a] = q->aabb_min[a];
		g.rext[a] = q->aabb_max[a] - q->aabb_min[a];
		g.tmin[a] = q->train_aabb_min[a];
		g.tmax[a] = q->train_aabb_max[a];
	}
	return g;
}

extern "C" NsbStatus nsb_density_on_grid(NsbContext* c, const NsbGridQuery* q, float* density_dev, void* stream) {
	if (!c || !q || !density_dev) return fail(NSB_ERR_INVALID, "null argument");
	if (!c->has_model) return fail(NSB_ERR_STATE, "nsb_density_on_grid: nsb_upload_model has not been called");
	if (!c->d_density_grid.get()) return fail(NSB_ERR_STATE, "nsb_density_on_grid: no density grid (nsb_upload_density_grid or nsb_update_density_grid)");
	if (!grid_res_ok(q->res)) return fail(NSB_ERR_INVALID, "nsb_density_on_grid: res must be positive multiples of 16 with a 32-bit point count");
	CU(cudaSetDevice(c->device));
	const mesh::GridQuery g = grid_query(q);
	const uint64_t n = (uint64_t)g.res[0] * g.res[1] * g.res[2];
	(c->acc16 ? mesh::k_density_on_grid<true> : mesh::k_density_on_grid<false>)<<<tile_ctas(c, n, c->inference_ctas_per_sm), 128, sizeof(tc::TileSmem), (cudaStream_t)stream>>>(
		c->model, g, c->d_density_grid.get(), density_dev);
	CU(cudaGetLastError());
	return NSB_OK;
}

extern "C" NsbStatus nsb_marching_cubes(NsbContext* c, const float* density_dev, const int32_t* res, const float* aabb_min, const float* aabb_max, float thresh,
                                        uint64_t* n_vertices, uint64_t* n_indices, void* stream_) {
	if (!c || !density_dev || !res || !aabb_min || !aabb_max) return fail(NSB_ERR_INVALID, "null argument");
	if (!grid_res_ok(res)) return fail(NSB_ERR_INVALID, "nsb_marching_cubes: res must be positive multiples of 16 with a 32-bit point count");
	CU(cudaSetDevice(c->device));
	cudaStream_t st = (cudaStream_t)stream_;
	c->has_mesh = c->mesh_shaded = c->mesh_csr = c->mesh_normals_ok = false;
	c->opt_fresh = true;  // Testbed::marching_cubes creates a fresh optimiser (testbed_nerf.cu:4638-4645)
	c->mesh_nv = c->mesh_ni = 0;
	mesh::McGrid g;
	g.d = density_dev;
	g.rx = (uint32_t)res[0]; g.ry = (uint32_t)res[1]; g.rz = (uint32_t)res[2];
	g.rxy = g.rx * g.ry;
	g.n = g.rxy * g.rz;
	g.thresh = thresh;
	const uint32_t n_tiles = (g.n + mesh::TILE - 1) / mesh::TILE;
	CU(c->mc_tiles.reserve(2 * (size_t)n_tiles));
	CU(c->mc_voff.reserve(g.n));
	CU(c->mc_totals.reserve(2));
	uint32_t* tile_nv = c->mc_tiles.get();
	uint32_t* tile_nt = c->mc_tiles.get() + n_tiles;
	mesh::k_mc_count<<<n_tiles, mesh::THREADS, 0, st>>>(g, tile_nv, tile_nt);
	mesh::k_mc_scan<<<1, 512, 0, st>>>(n_tiles, tile_nv, tile_nt, c->mc_totals.get());
	CU(cudaGetLastError());
	unsigned long long tot[2];
	CU(cudaMemcpyAsync(tot, c->mc_totals.get(), sizeof(tot), cudaMemcpyDeviceToHost, st));
	CU(cudaStreamSynchronize(st));  // the one synchronisation: the sizes of the outputs (marching_cubes.cu:747-749)
	const uint64_t rows = (tot[0] + 127ull) & ~127ull;
	if (rows > 0xffffffffull || 3ull * tot[1] > 0xffffffffull)
		return fail(NSB_ERR_INVALID, "nsb_marching_cubes: %llu vertices / %llu triangles do not fit 32-bit indices", tot[0], tot[1]);
	CU(c->mesh_verts.reserve(3 * rows));
	CU(c->mesh_idx.reserve(3 * tot[1]));
	if (rows) CU(cudaMemsetAsync(c->mesh_verts.get(), 0, 3 * rows * sizeof(float), st));  // verts_out.memset(0): the padding rows sit at the origin
	float sc[3];
	for (int a = 0; a < 3; ++a) sc[a] = (aabb_max[a] - aabb_min[a]) / (float)res[a];  // (aabb.max - aabb.min).cwiseQuotient(res_3d) (:224)
	mesh::k_mc_vertices<<<n_tiles, mesh::THREADS, 0, st>>>(g, tile_nv, sc[0], sc[1], sc[2], aabb_min[0], aabb_min[1], aabb_min[2], c->mc_voff.get(), c->mesh_verts.get());
	mesh::k_mc_faces<<<n_tiles, mesh::THREADS, 0, st>>>(g, tile_nt, c->mc_voff.get(), c->mesh_idx.get());
	CU(cudaGetLastError());
	c->mesh_nv = tot[0];
	c->mesh_ni = 3 * tot[1];
	c->has_mesh = true;
	if (n_vertices) *n_vertices = c->mesh_nv;
	if (n_indices) *n_indices = c->mesh_ni;
	return NSB_OK;
}

// The per-vertex triangle lists of the current mesh, built once per mesh: degrees, their exclusive scan, then the triangle ids per vertex
// (in slot order; the kernels that read a list visit it sorted)
static NsbStatus mesh_build_csr(NsbContext* c, cudaStream_t st) {
	if (c->mesh_csr) return NSB_OK;
	const uint32_t nv = (uint32_t)c->mesh_nv, nt = (uint32_t)(c->mesh_ni / 3);
	CU(c->mesh_start.reserve((size_t)nv + 1));
	CU(c->mesh_cursor.reserve((size_t)nv + 1));
	CU(c->mesh_adj.reserve(nt ? (size_t)3 * nt : 1));
	size_t tmp_bytes = 0;
	CU(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, c->mesh_cursor.get(), c->mesh_start.get(), nv + 1, st));
	CU(c->mesh_scan_tmp.reserve(tmp_bytes));
	CU(cudaMemsetAsync(c->mesh_cursor.get(), 0, ((size_t)nv + 1) * 4, st));
	if (nt) mesh::k_mesh_degree<<<(nt + 255) / 256, 256, 0, st>>>(nt, c->mesh_idx.get(), c->mesh_cursor.get());
	CU(cub::DeviceScan::ExclusiveSum(c->mesh_scan_tmp.get(), tmp_bytes, c->mesh_cursor.get(), c->mesh_start.get(), nv + 1, st));
	CU(cudaMemsetAsync(c->mesh_cursor.get(), 0, ((size_t)nv + 1) * 4, st));
	if (nt) mesh::k_mesh_fill<<<(nt + 255) / 256, 256, 0, st>>>(nt, c->mesh_idx.get(), c->mesh_start.get(), c->mesh_cursor.get(), c->mesh_adj.get());
	CU(cudaGetLastError());
	c->mesh_csr = true;
	return NSB_OK;
}

extern "C" NsbStatus nsb_mesh_shade(NsbContext* c, const float* train_aabb_min, const float* train_aabb_max, int32_t rgb_activation, int32_t linear_colors, void* stream_) {
	if (!c || !train_aabb_min || !train_aabb_max) return fail(NSB_ERR_INVALID, "null argument");
	if (!c->has_model) return fail(NSB_ERR_STATE, "nsb_mesh_shade: nsb_upload_model has not been called");
	if (!c->has_mesh) return fail(NSB_ERR_STATE, "nsb_mesh_shade: no mesh (nsb_marching_cubes)");
	if (rgb_activation < NSB_ACT_NONE || rgb_activation > NSB_ACT_EXPONENTIAL) return fail(NSB_ERR_INVALID, "nsb_mesh_shade: bad rgb_activation");
	CU(cudaSetDevice(c->device));
	cudaStream_t st = (cudaStream_t)stream_;
	const uint32_t nv = (uint32_t)c->mesh_nv, rows = (uint32_t)((c->mesh_nv + 127ull) & ~127ull);
	c->mesh_shaded = false;
	if (rows == 0) { c->mesh_shaded = c->mesh_normals_ok = true; return NSB_OK; }
	CU(c->mesh_normals.reserve(3 * (size_t)rows));
	CU(c->mesh_colors.reserve(3 * (size_t)rows));
	const NsbStatus csr = mesh_build_csr(c, st);
	if (csr != NSB_OK) return csr;
	mesh::k_mesh_normals<<<(rows + 255) / 256, 256, 0, st>>>(nv, rows, c->mesh_verts.get(), c->mesh_idx.get(), c->mesh_start.get(), c->mesh_adj.get(),
	                                                        c->mesh_normals.get());
	mesh::Aabb train;
	for (int a = 0; a < 3; ++a) { train.mn[a] = train_aabb_min[a]; train.mx[a] = train_aabb_max[a]; }
	(c->acc16 ? mesh::k_mesh_colors<true> : mesh::k_mesh_colors<false>)<<<tile_ctas(c, rows, c->inference_ctas_per_sm), 128, sizeof(tc::TileSmem), st>>>(
		c->model, rows, c->mesh_verts.get(), train, rgb_activation, linear_colors ? 1 : 0, c->mesh_colors.get());
	CU(cudaGetLastError());
	c->mesh_shaded = c->mesh_normals_ok = true;
	return NSB_OK;
}

extern "C" NsbStatus nsb_mesh_download(NsbContext* c, float* vertices, float* normals, float* colors, uint64_t vertex_rows, uint32_t* indices,
                                       uint64_t index_capacity) {
	if (!c) return fail(NSB_ERR_INVALID, "null context");
	if (!c->has_mesh) return fail(NSB_ERR_STATE, "nsb_mesh_download: no mesh (nsb_marching_cubes)");
	const uint64_t rows = (c->mesh_nv + 127ull) & ~127ull;
	if ((vertices || normals || colors) && vertex_rows > rows)
		return fail(NSB_ERR_INVALID, "nsb_mesh_download: %llu vertex rows asked, the mesh has %llu (%llu vertices + padding)", (unsigned long long)vertex_rows,
		            (unsigned long long)rows, (unsigned long long)c->mesh_nv);
	if (indices && index_capacity < c->mesh_ni)
		return fail(NSB_ERR_INVALID, "nsb_mesh_download: index buffer too small (%llu needed)", (unsigned long long)c->mesh_ni);
	if ((normals && !c->mesh_normals_ok) || (colors && !c->mesh_shaded))
		return fail(NSB_ERR_STATE, "nsb_mesh_download: normals need nsb_mesh_shade or nsb_mesh_optimise, colours nsb_mesh_shade");
	CU(cudaSetDevice(c->device));
	CU(cudaDeviceSynchronize());
	if (vertex_rows) {
		if (vertices) CU(cudaMemcpy(vertices, c->mesh_verts.get(), 3 * vertex_rows * 4, cudaMemcpyDeviceToHost));
		if (normals) CU(cudaMemcpy(normals, c->mesh_normals.get(), 3 * vertex_rows * 4, cudaMemcpyDeviceToHost));
		if (colors) CU(cudaMemcpy(colors, c->mesh_colors.get(), 3 * vertex_rows * 4, cudaMemcpyDeviceToHost));
	}
	if (indices && c->mesh_ni) CU(cudaMemcpy(indices, c->mesh_idx.get(), c->mesh_ni * 4, cudaMemcpyDeviceToHost));
	return NSB_OK;
}

// ---- mesh optimisation (Testbed::optimise_mesh_step, testbed_nerf.cu:4470-4513) ---------------------------------------------
extern "C" NsbStatus nsb_density_gradient(NsbContext* c, const float* coords, uint32_t n, float* grad, uint32_t grad_stride_floats, uint16_t* density_fp16,
                                          uint16_t* dfeat_fp16, uint32_t n_padded, void* stream) {
	if (!c) return fail(NSB_ERR_INVALID, "null context");
	if (!c->has_model) return fail(NSB_ERR_STATE, "nsb_density_gradient: nsb_upload_model has not been called");
	if (n && (!coords || !grad)) return fail(NSB_ERR_INVALID, "nsb_density_gradient: null argument");
	if (grad_stride_floats < 3) return fail(NSB_ERR_INVALID, "nsb_density_gradient: grad_stride_floats < 3");
	if (n_padded < n) return fail(NSB_ERR_INVALID, "nsb_density_gradient: n_padded < n");
	if (n_padded == 0) return NSB_OK;
	CU(cudaSetDevice(c->device));
	meshopt::GradIo io{};
	io.in = coords; io.n = n; io.n_padded = n_padded;
	io.grad = grad; io.grad_stride = grad_stride_floats;
	io.dens = reinterpret_cast<__half*>(density_fp16); io.dfeat = reinterpret_cast<__half*>(dfeat_fp16);
	(c->acc16 ? meshopt::k_density_gradient<true, false> : meshopt::k_density_gradient<false, false>)<<<tile_ctas(c, n_padded, c->inference_ctas_per_sm), 128, sizeof(meshopt::GradSmem), (cudaStream_t)stream>>>(
		c->model, io);
	CU(cudaGetLastError());
	return NSB_OK;
}

extern "C" NsbStatus nsb_mesh_optimise(NsbContext* c, const NsbMeshOptimise* p, uint32_t n_steps, void* stream_) {
	if (!c || !p) return fail(NSB_ERR_INVALID, "null argument");
	if (!c->has_model) return fail(NSB_ERR_STATE, "nsb_mesh_optimise: nsb_upload_model has not been called");
	if (!c->has_mesh) return fail(NSB_ERR_STATE, "nsb_mesh_optimise: no mesh (nsb_marching_cubes)");
	const uint32_t nv = (uint32_t)c->mesh_nv, rows = (uint32_t)((c->mesh_nv + 127ull) & ~127ull);
	if (rows == 0) { c->mesh_normals_ok = true; return NSB_OK; }  // an empty mesh has no normals to compute, as in nsb_mesh_shade
	if (n_steps == 0) return NSB_OK;
	CU(cudaSetDevice(c->device));
	cudaStream_t st = (cudaStream_t)stream_;
	const NsbStatus csr = mesh_build_csr(c, st);
	if (csr != NSB_OK) return csr;
	const size_t n3 = 3 * (size_t)rows;
	CU(c->mesh_normals.reserve(n3));
	if (c->opt_fresh || c->opt_m1.capacity() < n3) {
		CU(c->opt_pos.reserve(n3));
		CU(c->opt_m1.reserve(n3));
		CU(c->opt_m2.reserve(n3));
		CU(c->opt_steps.reserve(n3));
		CU(c->opt_grad.reserve(n3));
		CU(c->opt_dens.reserve(rows));
		CU(cudaMemsetAsync(c->opt_m1.get(), 0, n3 * sizeof(float), st));
		CU(cudaMemsetAsync(c->opt_m2.get(), 0, n3 * sizeof(float), st));
		CU(cudaMemsetAsync(c->opt_steps.get(), 0, n3 * sizeof(uint32_t), st));
		c->opt_fresh = false;
	}
	meshopt::GradIo io{};
	io.n = rows; io.n_padded = rows;
	io.grad_stride = 3;
	io.dens = c->opt_dens.get();
	io.dfeat = nullptr;
	for (int a = 0; a < 3; ++a) { io.train.mn[a] = p->train_aabb_min[a]; io.train.mx[a] = p->train_aabb_max[a]; }
	const meshopt::OptParams op{p->thresh, p->smooth_amount, p->density_amount, p->inflate_amount};
	const uint32_t grid = tile_ctas(c, rows, c->inference_ctas_per_sm);
	auto grad_kernel = c->acc16 ? meshopt::k_density_gradient<true, true> : meshopt::k_density_gradient<false, true>;
	for (uint32_t s = 0; s < n_steps; ++s) {
		io.in = c->mesh_verts.get();
		io.grad = c->opt_grad.get();
		grad_kernel<<<grid, 128, sizeof(meshopt::GradSmem), st>>>(c->model, io);
		meshopt::k_mesh_opt_step<<<(rows + 255) / 256, 256, 0, st>>>(nv, rows, c->mesh_verts.get(), c->opt_pos.get(), c->mesh_idx.get(), c->mesh_start.get(),
		                                                            c->mesh_adj.get(), c->opt_dens.get(), c->opt_grad.get(), op, c->opt_m1.get(), c->opt_m2.get(),
		                                                            c->opt_steps.get(), c->mesh_normals.get());
		CU(cudaGetLastError());
		std::swap(c->mesh_verts, c->opt_pos);  // the new positions become the mesh; the old buffer is the next step's output
	}
	c->mesh_normals_ok = true;
	return NSB_OK;
}

// ---- density and RGBA slices (the export panel's "Save density PNG" / "Save RGBA PNG sequence", testbed.cu:952-966) ---------------
static bool act_ok(int32_t a) { return a >= NSB_ACT_NONE && a <= NSB_ACT_EXPONENTIAL; }

extern "C" NsbStatus nsb_rgba_on_grid(NsbContext* c, const NsbGridQuery* q, const float* ray_dir, int32_t rgb_activation, int32_t density_activation,
                                      float* rgba_dev, void* stream) {
	if (!c || !q || !ray_dir || !rgba_dev) return fail(NSB_ERR_INVALID, "null argument");
	if (!c->has_model) return fail(NSB_ERR_STATE, "nsb_rgba_on_grid: nsb_upload_model has not been called");
	if (!grid_res_ok(q->res)) return fail(NSB_ERR_INVALID, "nsb_rgba_on_grid: res must be positive multiples of 16 with a 32-bit point count");
	if (!act_ok(rgb_activation) || !act_ok(density_activation)) return fail(NSB_ERR_INVALID, "nsb_rgba_on_grid: bad activation");
	if ((uintptr_t)rgba_dev & 15u) return fail(NSB_ERR_INVALID, "nsb_rgba_on_grid: rgba_dev must be 16-byte aligned");
	CU(cudaSetDevice(c->device));
	const mesh::GridQuery g = grid_query(q);
	const uint64_t n = (uint64_t)g.res[0] * g.res[1] * g.res[2];
	(c->acc16 ? slices::k_rgba_on_grid<true> : slices::k_rgba_on_grid<false>)<<<tile_ctas(c, n, c->inference_ctas_per_sm), 128, sizeof(tc::TileSmem), (cudaStream_t)stream>>>(
		c->model, g, ray_dir[0], ray_dir[1], ray_dir[2], rgb_activation, density_activation, reinterpret_cast<float4*>(rgba_dev));
	CU(cudaGetLastError());
	return NSB_OK;
}

// the grid and its images after the optional y/z swap (marching_cubes.cu:938-945, :984-989); false unless every res is positive, the point
// count fits 32 bits and the mosaic's width and height fit 32 bits
static bool slices_of(const int32_t* res, int32_t swap_y_z, slices::Slices* s, uint32_t* w, uint32_t* h) {
	if (!res || res[0] <= 0 || res[1] <= 0 || res[2] <= 0) return false;
	if ((uint64_t)res[0] * (uint64_t)res[1] * (uint64_t)res[2] > 0xffffffffull) return false;
	s->rx = (uint32_t)res[0]; s->ry = (uint32_t)res[1]; s->rz = (uint32_t)res[2];
	s->swap = swap_y_z ? 1u : 0u;
	s->sy = swap_y_z ? s->rz : s->ry;
	s->sz = swap_y_z ? s->ry : s->rz;
	const uint32_t ndown = (uint32_t)sqrtf((float)s->sz);
	const uint32_t nacross = (s->sz + ndown - 1) / ndown;
	const uint64_t ww = (uint64_t)s->rx * nacross, hh = (uint64_t)s->sy * ndown;
	if (ww > 0xffffffffull || hh > 0xffffffffull) return false;
	*w = (uint32_t)ww;
	*h = (uint32_t)hh;
	return true;
}

extern "C" NsbStatus nsb_density_png_extent(const int32_t* res, int32_t swap_y_z, uint32_t* w, uint32_t* h) {
	if (!res || !w || !h) return fail(NSB_ERR_INVALID, "null argument");
	slices::Slices s;
	if (!slices_of(res, swap_y_z, &s, w, h)) return fail(NSB_ERR_INVALID, "nsb_density_png_extent: res must be positive with a 32-bit point count");
	return NSB_OK;
}

static uint32_t slice_ctas(const NsbContext* c, uint64_t n) {
	const uint64_t grid = (n + 255) / 256, cap = (uint64_t)c->sm_count * 8;
	return (uint32_t)(grid < 1 ? 1 : (grid > cap ? cap : grid));
}

extern "C" NsbStatus nsb_density_png(NsbContext* c, const float* density_dev, const int32_t* res, float thresh, float density_range, int32_t swap_y_z,
                                     uint8_t* pixels_dev, uint64_t* counts_dev, void* stream) {
	if (!c || !density_dev || !res || !pixels_dev || !counts_dev) return fail(NSB_ERR_INVALID, "null argument");
	slices::Slices s;
	uint32_t w, h;
	if (!slices_of(res, swap_y_z, &s, &w, &h)) return fail(NSB_ERR_INVALID, "nsb_density_png: res must be positive with a 32-bit point count");
	if (!(density_range > 0.0f) || !std::isfinite(density_range)) return fail(NSB_ERR_INVALID, "nsb_density_png: density_range must be positive and finite");
	CU(cudaSetDevice(c->device));
	cudaStream_t st = (cudaStream_t)stream;
	const uint32_t nacross = w / s.rx;
	const float scale = 128.f / density_range;  // density_scale (marching_cubes.cu:899)
	CU(cudaMemsetAsync(counts_dev, 0, 2 * sizeof(uint64_t), st));
	const uint64_t n_px = (uint64_t)w * h;
	slices::k_density_png<<<slice_ctas(c, n_px), 256, 0, st>>>(s, density_dev, thresh, scale, w, nacross, pixels_dev,
	                                                            reinterpret_cast<unsigned long long*>(counts_dev));
	CU(cudaGetLastError());
	return NSB_OK;
}

extern "C" NsbStatus nsb_rgba_png(NsbContext* c, const float* rgba_dev, const int32_t* res, int32_t swap_y_z, uint8_t* pixels_dev, void* stream) {
	if (!c || !rgba_dev || !res || !pixels_dev) return fail(NSB_ERR_INVALID, "null argument");
	slices::Slices s;
	uint32_t w, h;
	if (!slices_of(res, swap_y_z, &s, &w, &h)) return fail(NSB_ERR_INVALID, "nsb_rgba_png: res must be positive with a 32-bit point count");
	if (((uintptr_t)rgba_dev & 15u) || ((uintptr_t)pixels_dev & 3u)) return fail(NSB_ERR_INVALID, "nsb_rgba_png: rgba_dev must be 16-byte, pixels_dev 4-byte aligned");
	CU(cudaSetDevice(c->device));
	slices::k_rgba_png<<<slice_ctas(c, (uint64_t)s.rx * s.ry * s.rz), 256, 0, (cudaStream_t)stream>>>(s, reinterpret_cast<const float4*>(rgba_dev),
	                                                                                                reinterpret_cast<uchar4*>(pixels_dev));
	CU(cudaGetLastError());
	return NSB_OK;
}
