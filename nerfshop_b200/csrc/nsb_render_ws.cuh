// nsb_render_ws.cuh — the warp-specialised form of the fused persistent renderer (frames without edit operators).
//
// k_render_fused lets every warp do everything: march -> 128 gathers -> five MMA layers (tile-wide barriers) -> composite, serially,
// per round. Here the two halves of a round run concurrently on different warps of ONE 768-thread CTA per SM (an experiment, opt-in NSB_WS=1):
//
//   producers (16 warps = 4 tiles x 128 ray slots): own the rays' march state. Per generation: learn which of their rays the consumers
//       terminated, refill free slots (same warp-coherent policy as the fused kernel), walk the occupancy grid to the next sample, gather the
//       32 hash-grid features straight into the first layer's wgmma A operand in shared memory, publish {t, flags, pixel} and arrive on the
//       tile's `full` mbarrier. They never wait for a tile barrier or an MMA.
//   consumers (8 warps = 2 warpgroups x 128 rows, each group serves two producer tiles alternately): wait for `full`, run the five wgmma
//       layers (first layer reads the producers' operand in place), composite the sample into the ray's accumulators, shade finished rays,
//       record terminations, and arrive on `empty`.
//
// A producer is at most one generation ahead of its consumer, so a ray that saturates costs one speculative sample (the consumer ignores
// it); rays that leave the AABB cost none. Per-ray results are unchanged: the same samples in the same order through the same device
// functions — all parity tests apply to this kernel unchanged.
#pragma once

namespace ws {

#ifndef NSB_WS_PT
#define NSB_WS_PT 4
#endif
#ifndef NSB_WS_CG
#define NSB_WS_CG 2
#endif
constexpr int PT = NSB_WS_PT;         // producer tiles (128 ray slots each)
constexpr int CG = NSB_WS_CG;         // consumer groups (128 threads each)
constexpr int TPG = PT / CG;          // producer tiles per consumer group
constexpr int THREADS = (PT + CG) * 128;
static_assert(PT == 2 * CG, "a consumer group serves TWO producer tiles");

enum { F_SAMPLE = 1u, F_FIRST = 2u, F_EXIT = 4u, F_DROP = 8u };
enum { S_PX = 0, S_PY, S_PZ, S_DT, S_DX, S_DY, S_DZ, S_FLAGS, S_FIELDS };  // per sample: warped position, warped dt, warped direction, flags (F_FIRST: S_DT holds the pixel)
// consumer-side ray state, parked in shared memory between generations (a group alternates between two tiles)
enum { A_CR = 0, A_CG, A_CB, A_CA, A_DEPTH, A_MAXW, A_PIX, A_META, A_FIELDS };  // META: bit 31 alive, low bits n_steps

struct __align__(128) Tile {  // the wgmma descriptors address feat in 16-byte units
	uint8_t feat[tc::A32_BYTES];           // ONE operand buffer: released (feat_free) as soon as the first layer's MMAs have completed, long before the generation is done
	uint32_t out[3][128];                  // network outputs the composite needs: density raw | (r, g) | (b, -) as packed fp16
	uint64_t feat_free;
	uint32_t side[2][S_FIELDS][128];
	float acc[A_FIELDS][128];
	uint32_t died_epoch[128];
	uint32_t fin[2][4];
	uint64_t full[2], empty[2];
	uint32_t stop, epoch_pad[3];
	uint32_t cepoch[128];  // consumer's ray counter per slot
};
struct __align__(128) Group {
	uint8_t a64[tc::A64_BYTES];  // the group's operand space (rgb-network input, output hand-back)
};
struct __align__(128) Smem {
	uint8_t w[tc::W_BYTES];
	Tile tile[PT];
	Group grp[CG];
	uint64_t w_bar;
	uint32_t pad[2];
};

}  // namespace ws

__global__ void __launch_bounds__(ws::THREADS, 1) k_render_ws(const DevFrame f, const DevModel m, const uint8_t* __restrict__ bitfield, float4* __restrict__ fb,
                                                              float* __restrict__ depth_out, const RayRec* __restrict__ list, const uint32_t* __restrict__ n_queued_ptr,
                                                              uint32_t* fetch_counter, unsigned long long* __restrict__ stats, const int refill_thr, const int dda_budget) {
	using namespace ws;
	extern __shared__ __align__(128) uint8_t smem_raw[];
	Smem& S = *reinterpret_cast<Smem*>(smem_raw);
	const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
	const uint32_t n_queued = *n_queued_ptr;
	if (blockIdx.x * 128u * PT >= n_queued && blockIdx.x > 0) return;  // nothing this CTA could ever fetch

	if (threadIdx.x == 0) {
		for (int t = 0; t < PT; ++t) {
			for (int b = 0; b < 2; ++b) { tc::mbar_init(&S.tile[t].full[b], 4); tc::mbar_init(&S.tile[t].empty[b], 4); }
			tc::mbar_init(&S.tile[t].feat_free, 1);
			S.tile[t].stop = 0;
		}
		tc::fence_mbar_init();
	}
	for (uint32_t i = threadIdx.x; i < PT * 128u; i += THREADS) {
		S.tile[i >> 7].died_epoch[i & 127u] = 0u;
		S.tile[i >> 7].cepoch[i & 127u] = 0u;
		S.tile[i >> 7].acc[A_META][i & 127u] = __uint_as_float(0u);
	}
	tc::load_weights(S.w, &S.w_bar, m.w_image);
	__syncthreads();

	uint32_t c_hit = 0, c_samples = 0, n_gen = 0;
#ifdef NSB_PROFILE
	long long cyc_wait = 0, cyc_work = 0;  // producer: waiting on `empty` / marching + gathering; consumer: waiting on `full` / MLP + composite
#endif

	if (warp >= CG * 4u) {
		// =============================================== producer ===============================================
		const uint32_t pt = (warp - CG * 4u) >> 2, wt = (warp - CG * 4u) & 3u;  // tile, warp within the tile
		Tile& TL = S.tile[pt];
		const uint32_t slot = wt * 32u + lane;
		bool alive = false, exhausted = false;
		uint32_t ch_next = 0, ch_end = 0, pix = 0, n_steps = 0, epoch = 0;
		V3 ro = v3(0, 0, 0), rd = v3(0, 0, 1);
		float t = 0.0f;
		for (uint32_t g = 0;; ++g) {
			const uint32_t b = g & 1u;
#ifdef NSB_PROFILE
			const long long p0 = clock64();
#endif
			if (g >= 2) tc::mbar_wait_backoff(&TL.empty[b], ((g >> 1) - 1u) & 1u, 200);  // the consumer is done with generation g - 2 (this buffer)
#ifdef NSB_PROFILE
			const long long p1 = clock64();
			cyc_wait += p1 - p0;
#endif
			if (*reinterpret_cast<volatile uint32_t*>(&TL.stop)) break;
			if (alive && *reinterpret_cast<volatile uint32_t*>(&TL.died_epoch[slot]) == epoch) alive = false;  // saturated at the consumer
			// out of rays BEFORE this generation: everything this warp publishes from now on is empty (a generation that carries a last
			// F_EXIT / F_SAMPLE record must still be processed by the consumer, so the flag is taken at the top)
			const bool warp_done = exhausted && __ballot_sync(0xffffffffu, alive) == 0u;
			uint32_t flags = 0;
			{   // refill: same warp-convergent policy as k_render_fused (consecutive queue entries = neighbouring pixels)
				const unsigned alive_m = __ballot_sync(0xffffffffu, alive);
				const unsigned want = exhausted ? 0u : ~alive_m;
				if (want && __popc(alive_m) <= (refill_thr & 0xff)) {
					const uint32_t need = (uint32_t)__popc(want), rank = (uint32_t)__popc(want & ((1u << lane) - 1u));
					const uint32_t chunk = (uint32_t)refill_thr >> 8;
					uint32_t given = 0, qi = 0xffffffffu;
					while (given < need) {
						if (ch_next >= ch_end) {
							const uint32_t claim = chunk ? chunk : need - given;
							uint32_t base = 0;
							if (lane == 0) base = atomicAdd(fetch_counter, claim);
							base = __shfl_sync(0xffffffffu, base, 0);
							if (base >= n_queued) { exhausted = true; break; }
							ch_next = base;
							ch_end = min(base + claim, n_queued);
						}
						const uint32_t take = min(need - given, ch_end - ch_next);
						if (!alive && rank >= given && rank < given + take) qi = ch_next + (rank - given);
						ch_next += take;
						given += take;
					}
					if (qi != 0xffffffffu) {
						const RayRec rr = list[qi];
						pix = rr.pix;
						Ray r;
						make_ray(f, pix % (uint32_t)f.W, pix / (uint32_t)f.W, r);
						ro = r.o; rd = r.d;
						t = rr.t;
						n_steps = 0;
						alive = true;
						++epoch;
						flags |= F_FIRST;
					}
				}
			}
			bool has_sample = false;
			float dt = 0.0f;
			V3 pos = v3(0, 0, 0);
			{
				int budget = dda_budget;
				for (;;) {
					if (!alive) break;
					if (n_steps >= MARCH_ITER - 1) { alive = false; flags |= F_DROP; break; }  // still marching after MARCH_ITER steps: dropped (:2812)
					const V3 idir = v3(div_(1.0f, rd.x), div_(1.0f, rd.y), div_(1.0f, rd.z));
					const MarchResult mr = next_occupied_budget(f, bitfield, ro, rd, idir, t, dt, pos, budget);
					if (mr == MARCH_FOUND) { has_sample = true; break; }
					if (mr == MARCH_EXIT) { alive = false; flags |= F_EXIT; break; }
					break;  // MARCH_PENDING: resume next generation
				}
			}
			V3 pw = v3(0, 0, 0);
			if (has_sample) {
				t = add(t, dt);
				pw = warp_position(pos, f.tmin, f.tmax);
				++n_steps;
				flags |= F_SAMPLE;
			}
			if (g >= 1) tc::mbar_wait_backoff(&TL.feat_free, (g - 1u) & 1u, 50);  // the first layer of generation g - 1 has read the operand
			encode_to_a32(TL.feat, m, has_sample, pw, slot);
			if (flags & (F_SAMPLE | F_FIRST)) {
				const V3 dw = warp_direction(rd);
				TL.side[b][S_PX][slot] = __float_as_uint(pw.x); TL.side[b][S_PY][slot] = __float_as_uint(pw.y); TL.side[b][S_PZ][slot] = __float_as_uint(pw.z);
				TL.side[b][S_DX][slot] = __float_as_uint(dw.x); TL.side[b][S_DY][slot] = __float_as_uint(dw.y); TL.side[b][S_DZ][slot] = __float_as_uint(dw.z);
			}
			// a ray's first record carries its pixel in a separate word pair: a first record that is also a sample needs both dt and the pixel
			TL.side[b][S_DT][slot] = __float_as_uint(warp_dt(dt));
			TL.side[b][S_FLAGS][slot] = flags | ((flags & F_FIRST) ? (pix << 4) : 0u);
			tc::fence_async_smem();
			__syncwarp();
			if (lane == 0) {
				TL.fin[b][wt] = warp_done ? 1u : 0u;
				tc::mbar_arrive(&TL.full[b]);
			}
#ifdef NSB_PROFILE
			cyc_work += clock64() - p1;
#endif
		}
#ifdef NSB_PROFILE
		if (lane == 0 && wt == 0 && pt == 0) { atomicAdd(stats + ST_CYC_ACQUIRE, (unsigned long long)cyc_wait); atomicAdd(stats + ST_CYC_ENCODE, (unsigned long long)cyc_work); }
#endif
	} else {
		// =============================================== consumer ===============================================
		// A group (one warpgroup) runs the network for its two producer tiles one after the other; the first layer reads the producer's operand
		// in place and releases it (feat_free) as soon as every warp of the group has read it.
		const uint32_t grp = warp >> 2, row = threadIdx.x & 127u;
		Group& G = S.grp[grp];
		Tile& TA = S.tile[grp * TPG + 0];
		Tile& TB = S.tile[grp * TPG + 1];
		tc::mbar_wait(&S.w_bar, 0);
		tc::TileCtx C;
		C.a32 = G.a64; C.w_addr = tc::smem_u32(S.w); C.row = row; C.bar_id = 1 + grp;
		const float sat = 1.0f - f.min_T;
		const V3 cam_fwd = v3(f.cam1[6], f.cam1[7], f.cam1[8]);
		for (uint32_t g = 0;; ++g) {
			const uint32_t b = g & 1u;
#ifdef NSB_PROFILE
			const long long q0 = clock64();
#endif
			tc::mbar_wait_backoff(&TA.full[b], (g >> 1) & 1u, 100);
			tc::mbar_wait_backoff(&TB.full[b], (g >> 1) & 1u, 100);
#ifdef NSB_PROFILE
			const long long q1 = clock64();
			cyc_wait += q1 - q0;
#endif
			{
				const volatile uint32_t* fa = TA.fin[b];
				const volatile uint32_t* fbn = TB.fin[b];
				if (fa[0] + fa[1] + fa[2] + fa[3] + fbn[0] + fbn[1] + fbn[2] + fbn[3] == 8u) {  // both tiles out of rays: this and all later generations are empty
					if (row == 0) {
						*reinterpret_cast<volatile uint32_t*>(&TA.stop) = 1u; *reinterpret_cast<volatile uint32_t*>(&TB.stop) = 1u;
						tc::mbar_arrive(&TA.feat_free); tc::mbar_arrive(&TB.feat_free);  // no first layer this generation: release the producers that already wait for it
					}
					__syncwarp();
					if (lane == 0) { tc::mbar_arrive(&TA.empty[b]); tc::mbar_arrive(&TB.empty[b]); }
					break;
				}
			}
			if (row == 0) ++n_gen;
			// ---- the five layers, one tile after the other ----
#pragma unroll 1
			for (uint32_t k = 0; k < (uint32_t)TPG; ++k) {
				Tile& TL = S.tile[grp * TPG + k];
				const V3 dw = v3(__uint_as_float(TL.side[b][S_DX][row]), __uint_as_float(TL.side[b][S_DY][row]), __uint_as_float(TL.side[b][S_DZ][row]));
				uint32_t dens[8], rgbo[8];
				tc::run_network<false>(C, dw, false, dens, rgbo, tc::smem_u32(TL.feat), &TL.feat_free);
				TL.out[0][row] = dens[0];
				TL.out[1][row] = rgbo[0];
				TL.out[2][row] = rgbo[1];
			}
			// ---- composite (composite_kernel_nerf :750-955) + shade (shade_kernel_nerf :2464-2482), one tile after the other ----
#pragma unroll 1
			for (uint32_t k = 0; k < (uint32_t)TPG; ++k) {
				Tile& TL = S.tile[grp * TPG + k];
				const uint32_t fl = TL.side[b][S_FLAGS][row];
				const uint32_t flags = fl & 15u;
				uint32_t meta = __float_as_uint(TL.acc[A_META][row]);
				uint32_t pix = __float_as_uint(TL.acc[A_PIX][row]);
				bool fresh = false;
				if (flags & F_FIRST) {
					pix = fl >> 4;  // pixels < 2^28 (the launcher falls back to k_render_fused for larger frames)
					TL.acc[A_PIX][row] = __uint_as_float(pix);
					meta = 0x80000000u;
					TL.cepoch[row] = TL.cepoch[row] + 1u;
					fresh = true;
				}
				bool alive = (meta >> 31) != 0u;
				uint32_t n_steps = meta & 0x7fffffffu;
				const bool has_sample = alive && (flags & F_SAMPLE);
				float cr = 0.0f, cg = 0.0f, cb = 0.0f, ca = 0.0f, ray_depth = 0.0f, max_weight = 0.0f;
				if (!fresh) {
					cr = TL.acc[A_CR][row]; cg = TL.acc[A_CG][row]; cb = TL.acc[A_CB][row]; ca = TL.acc[A_CA][row];
					ray_depth = TL.acc[A_DEPTH][row]; max_weight = TL.acc[A_MAXW][row];
				}
				auto finish = [&](bool left_aabb, float r_, float g_, float b_, float a_) {
					alive = false;
					if (!(a_ > 0.001f)) return;
					++c_hit;
					float r = r_, gg = g_, bb = b_, a = a_;
					if (f.mode == NSB_RENDER_COST) {
						float col = (float)(n_steps + (left_aabb ? 1u : 0u)) / 128.0f;
						r = gg = bb = col;
						a = 1.0f;
					}
					if (!f.linear_colors && f.mode == NSB_RENDER_SHADE) { r = srgb_to_linear(r); gg = srgb_to_linear(gg); bb = srgb_to_linear(bb); }
					float4 prev = fb[pix];
					float om = 1.0f - a;
					fb[pix] = make_float4(__fmaf_rn(prev.x, om, r), __fmaf_rn(prev.y, om, gg), __fmaf_rn(prev.z, om, bb), __fmaf_rn(prev.w, om, a));
					if (a > 0.2f) depth_out[pix] = ray_depth;
				};
				if (has_sample) {
					++n_steps;
					++c_samples;
					const V3 pw = v3(__uint_as_float(TL.side[b][S_PX][row]), __uint_as_float(TL.side[b][S_PY][row]), __uint_as_float(TL.side[b][S_PZ][row]));
					const float dtw = __uint_as_float(TL.side[b][S_DT][row]);
					const uint32_t o0 = TL.out[0][row], o1 = TL.out[1][row], o2 = TL.out[2][row];
					const V3 cpos = unwarp_position(pw, f.tmin, f.tmax);
					const float T = 1.0f - ca;
					const float dtu = unwarp_dt(dtw);
					const float sigma = network_to_density(h_lo(o0), f.density_act);
					const float alpha = 1.0f - __expf(-sigma * dtu);
					const float weight = alpha * T;
					float rgb[3] = {network_to_rgb(h_lo(o1), f.rgb_act), network_to_rgb(h_hi(o1), f.rgb_act), network_to_rgb(h_lo(o2), f.rgb_act)};
					if (f.mode != NSB_RENDER_SHADE) {
						V3 ro = v3(f.cam1[9], f.cam1[10], f.cam1[11]);
						if (f.mode == NSB_RENDER_DEPTH || f.mode == NSB_RENDER_DISTANCE) {  // the ray origin (rolling shutter: per pixel), debug modes only
							Ray r;
							make_ray(f, pix % (uint32_t)f.W, pix / (uint32_t)f.W, r);
							ro = r.o;
						}
						if (f.mode == NSB_RENDER_AO) { rgb[0] = rgb[1] = rgb[2] = alpha; }
						else if (f.mode == NSB_RENDER_POSITIONS) { rgb[0] = (cpos.x - 0.5f) / 2.0f + 0.5f; rgb[1] = (cpos.y - 0.5f) / 2.0f + 0.5f; rgb[2] = (cpos.z - 0.5f) / 2.0f + 0.5f; }
						else if (f.mode == NSB_RENDER_DEPTH) { float z = dot3(cam_fwd, vsub(cpos, ro)) * f.depth_scale; rgb[0] = rgb[1] = rgb[2] = z; }
						else if (f.mode == NSB_RENDER_DISTANCE) { V3 q = vsub(cpos, ro); float z = sqrtf(dot3(q, q)) * f.depth_scale; rgb[0] = rgb[1] = rgb[2] = z; }
						else if (f.mode == NSB_RENDER_STEPSIZE) { float wdt = warp_dt(dtu); rgb[0] = rgb[1] = rgb[2] = wdt; }
					}
					cr = __fmaf_rn(rgb[0], weight, cr);
					cg = __fmaf_rn(rgb[1], weight, cg);
					cb = __fmaf_rn(rgb[2], weight, cb);
					ca += weight;
					if (weight > max_weight) {
						max_weight = weight;
						ray_depth = dot3(cam_fwd, vsub(cpos, v3(f.cam1[9], f.cam1[10], f.cam1[11])));
					}
					if (ca > sat) {
						const float a = ca;
						cr = __fdiv_rn(cr, a); cg = __fdiv_rn(cg, a); cb = __fdiv_rn(cb, a); ca = __fdiv_rn(ca, a);
						finish(false, cr, cg, cb, ca);
						TL.died_epoch[row] = TL.cepoch[row];  // tell the producer (it learns it two generations later at most)
					}
				}
				if (alive && (flags & F_EXIT)) finish(true, cr, cg, cb, ca);
				if (flags & F_DROP) alive = false;
				TL.acc[A_CR][row] = cr; TL.acc[A_CG][row] = cg; TL.acc[A_CB][row] = cb; TL.acc[A_CA][row] = ca;
				TL.acc[A_DEPTH][row] = ray_depth; TL.acc[A_MAXW][row] = max_weight;
				TL.acc[A_META][row] = __uint_as_float((alive ? 0x80000000u : 0u) | (n_steps & 0x7fffffffu));
				__syncwarp();
				if (lane == 0) tc::mbar_arrive(&TL.empty[b]);
			}
#ifdef NSB_PROFILE
			cyc_work += clock64() - q1;
#endif
		}
#ifdef NSB_PROFILE
		if (threadIdx.x == 0) { atomicAdd(stats + ST_CYC_MLP, (unsigned long long)cyc_wait); atomicAdd(stats + ST_CYC_COMPOSITE, (unsigned long long)cyc_work); }
#endif
	}

	if (threadIdx.x == 0) {
		atomicAdd(stats + ST_ROUNDS, (unsigned long long)n_gen);
		atomicAdd(stats + ST_CTAS, 1ull);
	}
	unsigned long long cnt[2] = {c_hit, c_samples};
	const int slot_id[2] = {ST_HIT, ST_SAMPLES};
#pragma unroll
	for (int k = 0; k < 2; ++k) {
		unsigned long long v = cnt[k];
		for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
		if (lane == 0 && v) atomicAdd(stats + slot_id[k], v);
	}
}
