/*
 * nerfshop_oracle.cpp — CPU restatement of NeRFshop's interactive render path.
 *
 * TEST INFRASTRUCTURE ONLY. Nothing in the product (nerfshop_b200/, include/) may
 * call, link or import this file; only tests/, __graft_entry__.smoke() and the
 * cpu_baseline / --impl reference legs of bench.py do, and only as the checker /
 * CPU baseline.
 *
 * PARITY: pinned to the reference's own code for everything that lives in /root/reference. oracle/ref_build.py compiles
 * the reference's sources for this path (Testbed::render_nerf, NerfTracer::trace / init_rays_from_camera, every kernel they
 * launch, the edit-operator kernels, update_density_grid_nerf_operator, accumulate / tonemap, mvc.h, svd3.h, build_tet_grid)
 * from where they lie into oracle/_ref/ (CPU build, and an nvcc build for the GPU tests) behind stand-ins for the absent
 * submodules; tests/test_oracle_vs_ref.py and tests/test_frame_extras_cpu.py hold this file to them (identical sample
 * streams, frames <= 6.5e-4, identical occupancy grids / bitfields / tet LUTs). The reference ships no tests, golden vectors or
 * fixtures of its own (SURVEY.md sections 4, 8c) and its build system cannot run here (tiny-cuda-nn, Eigen, ... are absent
 * submodules). STILL UNPINNED: the hash-grid / SH / fully-fused-MLP arithmetic, which lives in the un-vendored private fork
 * gitlab.inria.fr/cjambon/tcnn-pyngp.git@pyngp-api (commit unrecorded): those three ops restate the published tiny-cuda-nn
 * algorithm of that era (SURVEY.md Appendix B) with the accumulator rounding policy as an explicit switch (orc_set_mlp_policy).
 * The golden vectors under tests/golden/ are minted by this file (tests/golden/make_golden.py).
 *
 * Numerics contract (shared with the CUDA path, DESIGN.md §3): fp32 ops exactly as
 * written here, one rounding per operator, FMA only where fmaf() is spelled out
 * (those are the places nvcc's default -fmad=true contracts the reference's
 * expressions); compile with -ffp-contract=off. fp16 values are rounded to nearest
 * even at the points marked h(). Transcendentals (expf, powf) are not bit-pinned.
 */
#include "../include/nerfshop_b200.h"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>

#ifdef _OPENMP
#include <omp.h>
#endif

namespace {

// ----------------------------------------------------------------------------------------
// fp16 <-> fp32/fp64, round-to-nearest-even, software (no dependence on F16C)
// ----------------------------------------------------------------------------------------
inline uint16_t d2h_slow(double v);
inline uint16_t d2h(double v) {
	// fast path for results in the normal fp16 range: round the 52-bit mantissa to 10 bits, ties to even
	uint64_t bits;
	std::memcpy(&bits, &v, 8);
	int exp = (int)((bits >> 52) & 0x7ffu) - 1023;
	if (exp >= -14 && exp <= 14) {
		uint64_t mant = bits & ((1ull << 52) - 1);
		uint32_t m = (uint32_t)(mant >> 42);
		uint64_t rem = mant & ((1ull << 42) - 1), halfway = 1ull << 41;
		if (rem > halfway || (rem == halfway && (m & 1u))) ++m;
		if (m == 1024u) { m = 0; ++exp; }
		return (uint16_t)(((bits >> 48) & 0x8000u) | (uint32_t)((exp + 15) << 10) | m);
	}
	return d2h_slow(v);
}
inline uint16_t d2h_slow(double v) {
	uint16_t sign = std::signbit(v) ? 0x8000u : 0u;
	if (std::isnan(v)) return (uint16_t)(sign | 0x7e00u);
	double a = std::fabs(v);
	if (a >= 65520.0) return (uint16_t)(sign | 0x7c00u);
	if (a == 0.0) return sign;
	int e;
	std::frexp(a, &e); // a = m * 2^e, m in [0.5,1)
	int E = e - 1;     // a = 1.xxx * 2^E
	if (E >= -14) {
		double q = std::ldexp(a, 10 - E);      // in [1024, 2048)
		long r = (long)std::nearbyint(q);      // RN-even in the default rounding mode
		if (r == 2048) { r = 1024; ++E; }
		if (E > 15) return (uint16_t)(sign | 0x7c00u);
		return (uint16_t)(sign | (uint16_t)((E + 15) << 10) | (uint16_t)(r - 1024));
	}
	double q = std::ldexp(a, 24); // subnormal: units of 2^-24
	long r = (long)std::nearbyint(q);
	return (uint16_t)(sign | (uint16_t)r);
}
inline uint16_t f2h(float f) { return d2h((double)f); }
inline float h2f(uint16_t h) {
	uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
	uint32_t exp = (h >> 10) & 0x1fu;
	uint32_t man = h & 0x3ffu;
	float out;
	if (exp == 0) {
		out = std::ldexp((float)man, -24);
		uint32_t b; std::memcpy(&b, &out, 4); b |= sign; std::memcpy(&out, &b, 4);
		return out;
	}
	uint32_t bits;
	if (exp == 31) bits = sign | 0x7f800000u | (man << 13);
	else bits = sign | ((exp + 112u) << 23) | (man << 13);
	std::memcpy(&out, &bits, 4);
	return out;
}
// __hadd: exact sum, one rounding (the double sum of two halves is exact)
inline uint16_t hadd(uint16_t a, uint16_t b) { return d2h((double)h2f(a) + (double)h2f(b)); }

struct V3 { float x, y, z; };
inline V3 v3(float x, float y, float z) { return V3{x, y, z}; }
inline V3 operator-(V3 a, V3 b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
inline V3 operator+(V3 a, V3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
inline V3 operator*(float s, V3 a) { return v3(s * a.x, s * a.y, s * a.z); }
// Eigen a.dot(b) for 3-vectors: Eigen's unrolled reduction tree is x0*y0 + (x1*y1 + x2*y2) (Redux.h, redux_novec_unroller) and nvcc 12.9
// contracts it to fma(x0,y0, fma(x1,y1, x2*y2)) — read off the PTX/SASS of the reference's own kernels (oracle/_ref, nvcc build) and
// confirmed bit for bit on the GPU (tests/test_gpu_vs_ref_cuda.py). Round 1 had the opposite association.
inline float dot3(V3 a, V3 b) { return fmaf(a.x, b.x, fmaf(a.y, b.y, a.z * b.z)); }
// Eigen cross: (a.y*b.z - a.z*b.y, ...) ; nvcc contracts each as fma(a.y, b.z, -(a.z*b.y))
inline V3 cross3(V3 a, V3 b) {
	return v3(fmaf(a.y, b.z, -(a.z * b.y)), fmaf(a.z, b.x, -(a.x * b.z)), fmaf(a.x, b.y, -(a.y * b.x)));
}
inline V3 madd3(V3 d, float t, V3 o) { return v3(fmaf(d.x, t, o.x), fmaf(d.y, t, o.y), fmaf(d.z, t, o.z)); }

// ----------------------------------------------------------------------------------------
// constants — common_nerf.h:16-39
// ----------------------------------------------------------------------------------------
constexpr uint32_t GRIDSIZE = 128;
constexpr uint32_t GRIDVOL = 128u * 128u * 128u;
constexpr int CASCADES = 5;
constexpr float NEAR_DISTANCE = 0.05f;
constexpr float SQRT3F = 1.73205080757f;
inline float MIN_STEP() { return SQRT3F / 1024.0f; }
inline float MAX_STEP() { return MIN_STEP() * 16.0f * 1024.0f / 128.0f; }
constexpr uint32_t MARCH_ITER = 10000; // testbed_nerf.cu:56

inline float clampf(float v, float lo, float hi) { return v < lo ? lo : (hi < v ? hi : v); }
inline int clampi(int v, int lo, int hi) { return v < lo ? lo : (hi < v ? hi : v); }

// ----------------------------------------------------------------------------------------
// random_val.cuh:159-322 — Owen-scrambled Sobol (Burley 2019)
// ----------------------------------------------------------------------------------------
const uint32_t SOBOL_DIR1[32] = {
	0x80000000, 0xc0000000, 0xa0000000, 0xf0000000, 0x88000000, 0xcc000000, 0xaa000000, 0xff000000,
	0x80800000, 0xc0c00000, 0xa0a00000, 0xf0f00000, 0x88880000, 0xcccc0000, 0xaaaa0000, 0xffff0000,
	0x80008000, 0xc000c000, 0xa000a000, 0xf000f000, 0x88008800, 0xcc00cc00, 0xaa00aa00, 0xff00ff00,
	0x80808080, 0xc0c0c0c0, 0xa0a0a0a0, 0xf0f0f0f0, 0x88888888, 0xcccccccc, 0xaaaaaaaa, 0xffffffff,
};
inline uint32_t sobol(uint32_t index, uint32_t dim) { // random_val.cuh:159-211 (dims 0,1 are the ones the path uses)
	uint32_t X = 0;
	for (uint32_t bit = 0; bit < 32; ++bit) {
		uint32_t mask = (index >> bit) & 1u;
		uint32_t d = dim == 0 ? (0x80000000u >> bit) : SOBOL_DIR1[bit];
		X ^= mask * d;
	}
	return X;
}
inline uint32_t hash_combine(uint32_t seed, uint32_t v) { return seed ^ (v + (seed << 6) + (seed >> 2)); }
inline uint32_t reverse_bits(uint32_t x) {
	x = (((x & 0xaaaaaaaau) >> 1) | ((x & 0x55555555u) << 1));
	x = (((x & 0xccccccccu) >> 2) | ((x & 0x33333333u) << 2));
	x = (((x & 0xf0f0f0f0u) >> 4) | ((x & 0x0f0f0f0fu) << 4));
	x = (((x & 0xff00ff00u) >> 8) | ((x & 0x00ff00ffu) << 8));
	return ((x >> 16) | (x << 16));
}
inline uint32_t laine_karras_permutation(uint32_t x, uint32_t seed) {
	x += seed;
	x ^= x * 0x6c50b47cu;
	x ^= x * 0xb82f1e52u;
	x ^= x * 0xc7afe638u;
	x ^= x * 0x8d22f6e6u;
	return x;
}
inline uint32_t nested_uniform_scramble_base2(uint32_t x, uint32_t seed) {
	return reverse_bits(laine_karras_permutation(reverse_bits(x), seed));
}
inline float u32_to_unit(uint32_t x) { return (float)x * (float)(1.0 / 4294967296.0); }
inline float ld_random_val(uint32_t index, uint32_t seed) { // random_val.cuh:284-288, dim 0
	index = nested_uniform_scramble_base2(index, seed);
	return u32_to_unit(nested_uniform_scramble_base2(sobol(index, 0), hash_combine(seed, 0)));
}
inline void ld_random_val_2d(uint32_t index, uint32_t seed, float* out) { // :278-282
	index = nested_uniform_scramble_base2(index, seed);
	for (uint32_t i = 0; i < 2; ++i) out[i] = u32_to_unit(nested_uniform_scramble_base2(sobol(index, i), hash_combine(seed, i)));
}
inline float fractf_(float x) { return x - floorf(x); }
inline void ld_random_pixel_offset(uint32_t spp, float* off) { // :317-322
	float a[2], b[2];
	ld_random_val_2d(0, 0xdeadbeefu, a);
	ld_random_val_2d(spp, 0xdeadbeefu, b);
	off[0] = fractf_((0.5f - a[0]) + b[0]);
	off[1] = fractf_((0.5f - a[1]) + b[1]);
}

// ----------------------------------------------------------------------------------------
// bounding_box.cuh:180-238
// ----------------------------------------------------------------------------------------
struct Box { V3 mn, mx; };
inline bool box_contains(const Box& b, V3 p) {
	return p.x >= b.mn.x && p.x <= b.mx.x && p.y >= b.mn.y && p.y <= b.mx.y && p.z >= b.mn.z && p.z <= b.mx.z;
}
inline float box_ray_tmin(const Box& b, V3 o, V3 d) { // ray_intersect(...).x()
	const float FMAX = 3.402823466e+38f;
	float tmin = (b.mn.x - o.x) / d.x, tmax = (b.mx.x - o.x) / d.x;
	if (tmin > tmax) std::swap(tmin, tmax);
	float tymin = (b.mn.y - o.y) / d.y, tymax = (b.mx.y - o.y) / d.y;
	if (tymin > tymax) std::swap(tymin, tymax);
	if (tmin > tymax || tymin > tmax) return FMAX;
	if (tymin > tmin) tmin = tymin;
	if (tymax < tmax) tmax = tymax;
	float tzmin = (b.mn.z - o.z) / d.z, tzmax = (b.mx.z - o.z) / d.z;
	if (tzmin > tzmax) std::swap(tzmin, tzmax);
	if (tmin > tzmax || tzmin > tmax) return FMAX;
	if (tzmin > tmin) tmin = tzmin;
	return tmin;
}
inline Box mkbox(const float* mn, const float* mx) { return Box{v3(mn[0], mn[1], mn[2]), v3(mx[0], mx[1], mx[2])}; }

// ----------------------------------------------------------------------------------------
// common_nerf.cu:5-177
// ----------------------------------------------------------------------------------------
inline V3 warp_position(V3 p, const Box& aabb) { // :5-10 -> relative_pos (bounding_box.cuh:96-98)
	V3 dg = aabb.mx - aabb.mn;
	return v3((p.x - aabb.mn.x) / dg.x, (p.y - aabb.mn.y) / dg.y, (p.z - aabb.mn.z) / dg.z);
}
inline V3 unwarp_position(V3 p, const Box& aabb) { // :12-17
	V3 dg = aabb.mx - aabb.mn;
	return v3(fmaf(p.x, dg.x, aabb.mn.x), fmaf(p.y, dg.y, aabb.mn.y), fmaf(p.z, dg.z, aabb.mn.z));
}
inline V3 warp_direction(V3 d) { return v3((d.x + 1.0f) * 0.5f, (d.y + 1.0f) * 0.5f, (d.z + 1.0f) * 0.5f); } // :20-22
inline V3 unwarp_direction(V3 d) { return v3(fmaf(d.x, 2.0f, -1.0f), fmaf(d.y, 2.0f, -1.0f), fmaf(d.z, 2.0f, -1.0f)); } // :24-26
inline float warp_dt(float dt) { // :28-31
	float max_stepsize = MIN_STEP() * 16.0f;
	return (dt - MIN_STEP()) / (max_stepsize - MIN_STEP());
}
inline float unwarp_dt(float dt) { // :33-36
	float max_stepsize = MIN_STEP() * 16.0f;
	return fmaf(dt, (max_stepsize - MIN_STEP()), MIN_STEP());
}
inline float calc_dt(float t, float cone_angle) { return clampf(t * cone_angle, MIN_STEP(), MAX_STEP()); } // :89-91

inline float signf_(float x) { return copysignf(1.0f, x); }
inline float distance_to_next_voxel(V3 pos, V3 dir, V3 idir, uint32_t res) { // :93-101
	float fr = (float)res;
	V3 p = v3(fr * pos.x, fr * pos.y, fr * pos.z);
	float tx = (floorf(fmaf(0.5f, signf_(dir.x), p.x + 0.5f)) - p.x) * idir.x;
	float ty = (floorf(fmaf(0.5f, signf_(dir.y), p.y + 0.5f)) - p.y) * idir.y;
	float tz = (floorf(fmaf(0.5f, signf_(dir.z), p.z + 0.5f)) - p.z) * idir.z;
	float t = fminf(fminf(tx, ty), tz);
	return fmaxf(t / fr, 0.0f);
}
inline float advance_to_next_voxel(float t, float cone, V3 pos, V3 dir, V3 idir, uint32_t res) { // :103-115
	float t_target = t + distance_to_next_voxel(pos, dir, idir, res);
	do { t += calc_dt(t, cone); } while (t < t_target);
	return t;
}
inline uint32_t expand_bits(uint32_t v) { // tcnn::morton3D
	v = (v * 0x00010001u) & 0xFF0000FFu;
	v = (v * 0x00000101u) & 0x0F00F00Fu;
	v = (v * 0x00000011u) & 0xC30C30C3u;
	v = (v * 0x00000005u) & 0x49249249u;
	return v;
}
inline uint32_t morton3D(uint32_t x, uint32_t y, uint32_t z) { return expand_bits(x) | (expand_bits(y) << 1) | (expand_bits(z) << 2); }
inline uint32_t cascaded_grid_idx_at(V3 pos, uint32_t mip) { // :117-136
	float mip_scale = std::ldexp(1.0f, -(int)mip);
	float px = fmaf(pos.x - 0.5f, mip_scale, 0.5f);
	float py = fmaf(pos.y - 0.5f, mip_scale, 0.5f);
	float pz = fmaf(pos.z - 0.5f, mip_scale, 0.5f);
	int ix = (int)(px * (float)GRIDSIZE), iy = (int)(py * (float)GRIDSIZE), iz = (int)(pz * (float)GRIDSIZE);
	return morton3D((uint32_t)clampi(ix, 0, 127), (uint32_t)clampi(iy, 0, 127), (uint32_t)clampi(iz, 0, 127));
}
inline bool bitfield_at(uint32_t idx, uint32_t mip, const uint8_t* bf) { // :138-141,153-155
	return (bf[idx / 8 + (GRIDVOL * mip) / 8] & (1u << (idx % 8))) != 0;
}
inline int mip_from_pos(V3 pos) { // :163-168
	int exponent;
	float maxval = fmaxf(fmaxf(fabsf(pos.x - 0.5f), fabsf(pos.y - 0.5f)), fabsf(pos.z - 0.5f));
	std::frexp(maxval, &exponent); // frexp(0) -> exponent 0 (so the exact centre maps to mip 1, as in the reference)
	return std::min(CASCADES - 1, std::max(0, exponent + 1));
}
inline int mip_from_dt(float dt, V3 pos) { // :170-177
	int mip = mip_from_pos(pos);
	dt *= (float)(2 * GRIDSIZE);
	if (dt < 1.0f) return mip;
	int exponent;
	std::frexp(dt, &exponent);
	return std::min(CASCADES - 1, std::max(exponent, mip));
}
inline float logistic_(float x) { return 1.0f / (1.0f + expf(-x)); }
inline float network_to_rgb(float v, int act) { // :38-47
	switch (act) {
		case NSB_ACT_NONE: return v;
		case NSB_ACT_RELU: return v > 0.0f ? v : 0.0f;
		case NSB_ACT_LOGISTIC: return logistic_(v);
		case NSB_ACT_EXPONENTIAL: return expf(clampf(v, -10.0f, 10.0f));
	}
	return 0.0f;
}
inline float network_to_density(float v, int act) { // :57-66
	switch (act) {
		case NSB_ACT_NONE: return v;
		case NSB_ACT_RELU: return v > 0.0f ? v : 0.0f;
		case NSB_ACT_LOGISTIC: return logistic_(v);
		case NSB_ACT_EXPONENTIAL: return expf(v);
	}
	return 0.0f;
}
inline float srgb_to_linear(float s) { // common_device.cuh:31-37
	if (s <= 0.04045f) return s / 12.92f;
	return powf((s + 0.055f) / 1.055f, 2.4f);
}
inline void evaluate_sh9(const float* sh /*9x3 col-major*/, V3 d, float* rgb) { // common_nerf.cu:218-245
	float p[9];
	float z2 = d.z * d.z;
	p[0] = 0.2820947917738781f;
	p[2] = 0.4886025119029199f * d.z;
	p[6] = fmaf(0.9461746957575601f, z2, -0.3153915652525201f);
	float c0 = d.x, s0 = d.y;
	p[3] = -0.48860251190292f * c0;
	p[1] = -0.48860251190292f * s0;
	float tb = -1.092548430592079f * d.z;
	p[7] = tb * c0;
	p[5] = tb * s0;
	float c1 = fmaf(d.x, c0, -(d.y * s0));
	float s1 = fmaf(d.x, s0, d.y * c0);
	p[8] = 0.5462742152960395f * c1;
	p[4] = 0.5462742152960395f * s1;
	for (int c = 0; c < 3; ++c) {
		float acc = p[0] * sh[c * 9 + 0];
		for (int k = 1; k < 9; ++k) acc = fmaf(p[k], sh[c * 9 + k], acc);
		rgb[c] = acc;
	}
}

// ----------------------------------------------------------------------------------------
// tiny-cuda-nn restatement (SURVEY.md Appendix B) — hash grid, SH-4, fully fused MLP
// ----------------------------------------------------------------------------------------
struct Level { float scale; uint32_t res; uint32_t offset; uint32_t size; };
struct Model {
	NsbModelDesc desc;
	const uint16_t* params;
	const uint16_t* w[5];      // W1 [64x32], W2 [16x64], W3 [64x32], W4 [64x64], W5 [16x64] (row-major out x in)
	const uint16_t* grid;
	std::vector<Level> levels;
	std::vector<float> wf[5];  // the fp16 weights widened once (exact)
	uint64_t n_params;
};

inline uint32_t next_multiple(uint32_t v, uint32_t m) { return ((v + m - 1) / m) * m; }

// The float -> int conversion of tcnn's `(int)floorf(p)` on the GPU, cvt.rzi.s32.f32: truncation toward zero, NaN -> 0, values outside
// the int range saturate to INT_MIN / INT_MAX. A C++ cast is undefined there (|p| >= 2^31, +-inf, NaN), so the oracle spells it out.
inline int32_t cvt_rzi_s32(double v) {
	if (v != v) return 0;
	if (v >= 2147483648.0) return INT32_MAX;
	if (v <= -2147483648.0) return INT32_MIN;
	return (int32_t)v;
}

// The accepted descriptions: the configs/nerf/base.json topology, log2_hashmap_size 1..24, base_resolution >= 1, per_level_scale >= 1
// (not NaN), every level's scale below 2^32 (so that `(uint32_t)ceilf(scale) + 1` is defined and fits).
bool model_init(Model& m, const NsbModelDesc* d, const uint16_t* params, uint64_t n_params) {
	if (!d || d->n_features_per_level != 2 || d->n_neurons != 64 || d->n_hidden_density != 1 || d->n_hidden_rgb != 2 ||
	    d->sh_degree != 4 || d->n_levels == 0 || d->n_levels != 16 || d->log2_hashmap_size == 0 || d->log2_hashmap_size > 24 ||
	    d->base_resolution == 0 || !(d->per_level_scale >= 1.0f)) return false;
	m.desc = *d;
	m.levels.resize(d->n_levels);
	float l2s = log2f(d->per_level_scale);
	uint32_t offset = 0;  // at most 16 x 2^24 entries
	for (uint32_t l = 0; l < d->n_levels; ++l) {
		float scale = exp2f((float)l * l2s) * (float)d->base_resolution - 1.0f; // grid_scale
		if (!(scale < 4294967296.0f)) return false;
		uint32_t res = (uint32_t)ceilf(scale) + 1u;                               // grid_resolution
		uint32_t max_params = 0xffffffffu / 2;
		double dense = (double)res * res * res;
		uint32_t n = dense > (double)max_params ? max_params : (uint32_t)dense;
		n = next_multiple(n, 8u);
		n = std::min(n, 1u << d->log2_hashmap_size);
		m.levels[l] = Level{scale, res, offset, n};
		offset += n;
	}
	uint64_t mlp = 64 * 32 + 16 * 64 + 64 * 32 + 64 * 64 + 16 * 64;
	m.n_params = mlp + (uint64_t)offset * 2;
	if (params) {
		if (n_params != m.n_params) return false;
		m.params = params;
		m.w[0] = params;
		m.w[1] = m.w[0] + 64 * 32;
		m.w[2] = m.w[1] + 16 * 64;
		m.w[3] = m.w[2] + 64 * 32;
		m.w[4] = m.w[3] + 64 * 64;
		m.grid = m.w[4] + 16 * 64;
		const int sizes[5] = {64 * 32, 16 * 64, 64 * 32, 64 * 64, 16 * 64};
		for (int i = 0; i < 5; ++i) {
			m.wf[i].resize(sizes[i]);
			for (int k = 0; k < sizes[i]; ++k) m.wf[i][k] = h2f(m.w[i][k]);
		}
	}
	return true;
}

// tcnn grid_index: the uint32 stride loop (it may wrap), hash where size < stride, then `index % size` on the uint32 index.
inline uint32_t grid_entry(const Level& L, const uint32_t* gl) {
	uint32_t stride = 1, index = 0;
	for (int dim = 0; dim < 3 && stride <= L.size; ++dim) { index += gl[dim] * stride; stride *= L.res; }
	if (L.size < stride) index = (gl[0] * 1u) ^ (gl[1] * 2654435761u) ^ (gl[2] * 805459861u);
	return index % L.size;
}

// tcnn kernel_grid<__half,3,2>, linear interpolation: out[l*2+f], fp16.
void encode_grid(const Model& m, V3 x, uint16_t* out /*32*/) {
	const float xin[3] = {x.x, x.y, x.z};
	for (uint32_t l = 0; l < m.desc.n_levels; ++l) {
		const Level& L = m.levels[l];
		float w[3];
		uint32_t g[3];
		for (int dim = 0; dim < 3; ++dim) { // pos_fract
			float p = fmaf(L.scale, xin[dim], 0.5f);
			float fl = floorf(p);
			g[dim] = (uint32_t)cvt_rzi_s32(fl);
			w[dim] = p - fl;
		}
		uint16_t acc[2] = {0, 0};
		for (uint32_t idx = 0; idx < 8; ++idx) {
			float weight = 1.0f;
			uint32_t gl[3];
			for (int dim = 0; dim < 3; ++dim) {
				if ((idx & (1u << dim)) == 0) { weight *= 1.0f - w[dim]; gl[dim] = g[dim]; }
				else { weight *= w[dim]; gl[dim] = g[dim] + 1u; }
			}
			const uint16_t* e = m.grid + ((uint64_t)L.offset + grid_entry(L, gl)) * 2;
			for (int f = 0; f < 2; ++f) acc[f] = hadd(acc[f], f2h(weight * h2f(e[f]))); // result += (T)(weight*data)
		}
		out[l * 2 + 0] = acc[0];
		out[l * 2 + 1] = acc[1];
	}
}

// tcnn SphericalHarmonics degree 4 on 2*d-1; fp16 out.
void encode_sh4(V3 dw, uint16_t* out /*16*/) {
	float x = fmaf(dw.x, 2.0f, -1.0f), y = fmaf(dw.y, 2.0f, -1.0f), z = fmaf(dw.z, 2.0f, -1.0f);
	float xy = x * y, xz = x * z, yz = y * z, x2 = x * x, y2 = y * y, z2 = z * z;
	float o[16];
	o[0] = 0.28209479177387814f;
	o[1] = -0.48860251190291987f * y;
	o[2] = 0.48860251190291987f * z;
	o[3] = -0.48860251190291987f * x;
	o[4] = 1.0925484305920792f * xy;
	o[5] = -1.0925484305920792f * yz;
	o[6] = 0.94617469575755997f * z2 - 0.31539156525251999f;
	o[7] = -1.0925484305920792f * xz;
	o[8] = 0.54627421529603959f * x2 - 0.54627421529603959f * y2;
	o[9] = (0.59004358992664352f * y) * (-3.0f * x2 + y2);
	o[10] = (2.8906114426405538f * xy) * z;
	o[11] = (0.45704579946446572f * y) * (1.0f - 5.0f * z2);
	o[12] = (0.3731763325901154f * z) * (5.0f * z2 - 3.0f);
	o[13] = (0.45704579946446572f * x) * (1.0f - 5.0f * z2);
	o[14] = (1.4453057213202769f * z) * (x2 - y2);
	o[15] = (0.59004358992664352f * x) * (-x2 + 3.0f * y2);
	for (int i = 0; i < 16; ++i) out[i] = f2h(o[i]);
}

// Accumulator policy of the fully fused MLPs (orc_set_mlp_policy):
//   1 (default) half accumulator fragments: tiny-cuda-nn's FullyFusedMLP of that era runs wmma m16n16k16 with __half accumulators (SURVEY.md
//     Appendix B; the submodule is absent, so unverifiable here): the running sum is rounded to fp16 after every k-chunk of 16 (products and
//     the 16-term partial sum inside one MMA are kept wide). The CUDA path's default (wgmma with an fp16 D) reproduces it 99.9 % bit for bit;
//   0 wide: every output is the exactly-rounded dot product (double accumulate, one rounding to fp16) — what fp32 accumulators
//     (NSB_MLP_ACC_F32) approximate to 2-4 fp16 ulps.
// tests/test_mlp_policy.py measures how far the two are apart in the framebuffer (up to 1e-2 on 0.02 % of the pixels).
int g_mlp_policy = 1;

// One fully-fused layer: y = W x, W [n_out x n_in] fp16 row-major, x fp16, y -> fp16.
void mlp_layer(const float* W, int n_out, int n_in, const uint16_t* x, bool relu, uint16_t* y) {
	double xf[64];
	for (int k = 0; k < n_in; ++k) xf[k] = (double)h2f(x[k]);
	for (int o = 0; o < n_out; ++o) {
		double acc = 0.0;
		const float* row = W + (size_t)o * n_in;
		if (g_mlp_policy == 1) {
			uint16_t acc_h = 0;
			for (int k0 = 0; k0 < n_in; k0 += 16) {
				double part = 0.0;
				for (int k = k0; k < k0 + 16 && k < n_in; ++k) part += (double)row[k] * xf[k];
				acc_h = d2h((double)h2f(acc_h) + part);
			}
			acc = (double)h2f(acc_h);
		} else {
			for (int k = 0; k < n_in; ++k) acc += (double)row[k] * xf[k];
		}
		float a = (float)acc;
		if (relu && !(a > 0.0f)) a = 0.0f;
		y[o] = f2h(a);
	}
}

// NerfNetworkFull::inference_mixed_precision_impl (nerf_network_full.h:62-96).
// density_out (16) optional; out16: rows 0-2 rgb raw, row 3 density raw, rows 4-15 rgb MLP padding outputs.
void network_forward(const Model& m, V3 pos_w, V3 dir_w, uint16_t* out16, uint16_t* density_out16, bool density_only) {
	uint16_t feat[32], h1[64], dout[16];
	encode_grid(m, pos_w, feat);
	mlp_layer(m.wf[0].data(), 64, 32, feat, true, h1);
	mlp_layer(m.wf[1].data(), 16, 64, h1, false, dout);
	if (density_out16) std::memcpy(density_out16, dout, 32);
	if (density_only) return;
	uint16_t rin[32], h2[64], h3[64];
	std::memcpy(rin, dout, 32);
	encode_sh4(dir_w, rin + 16);
	mlp_layer(m.wf[2].data(), 64, 32, rin, true, h2);
	mlp_layer(m.wf[3].data(), 64, 64, h2, true, h3);
	mlp_layer(m.wf[4].data(), 16, 64, h3, false, out16);
	out16[3] = dout[0]; // extract_density (nerf_network.h:42, nerf_network_full.h:89)
}

// ----------------------------------------------------------------------------------------
// editing — selection_utils.h:10-47, cage_deformation.cu:197-269,431-541, affine_duplication.cu:92-118
// ----------------------------------------------------------------------------------------
inline float scalar_tp(V3 a, V3 b, V3 c) { return dot3(a, cross3(b, c)); }
inline bool same_side_tet(V3 v1, V3 v2, V3 v3_, V3 v4, V3 p) {
	V3 normal = cross3(v2 - v1, v3_ - v1);
	float dotV4 = dot3(normal, v4 - v1);
	float dotP = dot3(normal, p - v1);
	return std::signbit(dotV4) == std::signbit(dotP);
}
inline bool point_in_tet(V3 a, V3 b, V3 c, V3 d, V3 p) {
	return same_side_tet(a, b, c, d, p) && same_side_tet(b, c, d, a, p) && same_side_tet(c, d, a, b, p) && same_side_tet(d, a, b, c, p);
}
inline void bary_tet(V3 a, V3 b, V3 c, V3 d, V3 p, float* out) {
	V3 vap = p - a, vbp = p - b, vab = b - a, vac = c - a, vad = d - a, vbc = c - b, vbd = d - b;
	float va6 = scalar_tp(vbp, vbd, vbc);
	float vb6 = scalar_tp(vap, vac, vad);
	float vc6 = scalar_tp(vap, vad, vab);
	float vd6 = scalar_tp(vap, vab, vac);
	float v6 = (float)(1.0 / (double)scalar_tp(vab, vac, vad)); // "1. / ..." is a double division in the reference
	out[0] = va6 * v6; out[1] = vb6 * v6; out[2] = vc6 * v6; out[3] = vd6 * v6;
}
inline V3 ldv(const float* p, uint32_t i) { return v3(p[3 * i], p[3 * i + 1], p[3 * i + 2]); }
inline V3 bary_mix(const float* b, V3 a0, V3 a1, V3 a2, V3 a3) { // ((b.x*a0 + b.y*a1) + b.z*a2) + b.w*a3; nvcc: fma(b3,a3, fma(b2,a2, fma(b0,a0, b1*a1)))
	return v3(fmaf(b[3], a3.x, fmaf(b[2], a2.x, fmaf(b[0], a0.x, b[1] * a1.x))),
	          fmaf(b[3], a3.y, fmaf(b[2], a2.y, fmaf(b[0], a0.y, b[1] * a1.y))),
	          fmaf(b[3], a3.z, fmaf(b[2], a2.z, fmaf(b[0], a0.z, b[1] * a1.z))));
}
inline V3 matvec3(const float* M /*col-major*/, V3 v) {
	return v3(fmaf(M[0], v.x, fmaf(M[3], v.y, M[6] * v.z)), fmaf(M[1], v.x, fmaf(M[4], v.y, M[7] * v.z)), fmaf(M[2], v.x, fmaf(M[5], v.y, M[8] * v.z)));  // row . v, Eigen tree
}
inline V3 matTvec3(const float* M /*col-major*/, V3 v) {
	return v3(fmaf(M[0], v.x, fmaf(M[1], v.y, M[2] * v.z)), fmaf(M[3], v.x, fmaf(M[4], v.y, M[5] * v.z)), fmaf(M[6], v.x, fmaf(M[7], v.y, M[8] * v.z)));
}

// find the first tet of `cell`'s candidate list that contains p (cage_deformation.cu:228-248)
inline int find_tet(const NsbEditOp& op, V3 p, float* bary) {
	int level = mip_from_pos(p);
	uint32_t cell = (uint32_t)level * GRIDVOL + cascaded_grid_idx_at(p, (uint32_t)level);
	for (uint32_t j = op.tet_lut_offsets[cell]; j < op.tet_lut_offsets[cell + 1]; ++j) {
		uint32_t t = op.tet_lut_idx[j];
		V3 a = ldv(op.vertices, op.tets[4 * t]), b = ldv(op.vertices, op.tets[4 * t + 1]);
		V3 c = ldv(op.vertices, op.tets[4 * t + 2]), d = ldv(op.vertices, op.tets[4 * t + 3]);
		if (point_in_tet(a, b, c, d, p)) { bary_tet(a, b, c, d, p, bary); return (int)t; }
	}
	return -1;
}

// interpolate_tet (cage_deformation.cu:197-269). pos/dir are the warped NerfCoordinate fields.
void cage_map(const NsbEditOp& op, V3& pos_w, V3& dir_w, bool& empty) {
	Box aabb = mkbox(op.scene_aabb_min, op.scene_aabb_max);
	Box dbox = mkbox(op.warped_bbox_min, op.warped_bbox_max);
	Box obox = mkbox(op.original_warped_bbox_min, op.original_warped_bbox_max);
	if (op.n_tets == 0) return; // map_rays early-out (cage_deformation.cu:549-551)
	bool in_deformed = false;
	if (box_contains(dbox, pos_w)) {
		V3 p = unwarp_position(pos_w, aabb);
		float b[4];
		int t = find_tet(op, p, b);
		if (t >= 0) {
			V3 canon = bary_mix(b, ldv(op.original_vertices, op.tets[4 * t]), ldv(op.original_vertices, op.tets[4 * t + 1]),
			                    ldv(op.original_vertices, op.tets[4 * t + 2]), ldv(op.original_vertices, op.tets[4 * t + 3]));
			pos_w = warp_position(canon, aabb);
			if (op.local_rotations) {
				V3 ud = unwarp_direction(dir_w);
				ud = matvec3(op.local_rotations + 9 * (size_t)t, ud);
				dir_w = warp_direction(ud);
			}
			in_deformed = true;
		}
	}
	if (!op.copy) {
		if (!in_deformed && box_contains(obox, pos_w)) {
			V3 p = unwarp_position(pos_w, aabb);
			int level = mip_from_pos(p);
			uint32_t idx = cascaded_grid_idx_at(p, (uint32_t)level);
			if (bitfield_at(idx, (uint32_t)level, op.original_bitfield)) empty = true;
		}
	}
}

inline bool abox_contains(const NsbAffineBox& b, V3 p) { // affine_bounding_box.cuh:88-93
	V3 mn = v3(b.min[0], b.min[1], b.min[2]);
	V3 u = v3(b.u[0], b.u[1], b.u[2]), v = v3(b.v[0], b.v[1], b.v[2]), w = v3(b.w[0], b.w[1], b.w[2]);
	V3 q = p - mn;
	float du = dot3(u, q), dv = dot3(v, q), dw = dot3(w, q);
	return du >= 0 && du < dot3(u, u) && dv >= 0 && dv < dot3(v, v) && dw >= 0 && dw < dot3(w, w);
}
// translate_in_box (affine_duplication.cu:92-118)
void affine_map(const NsbEditOp& op, V3& pos_w, V3& dir_w, bool& empty) {
	if (abox_contains(op.destination_box, pos_w)) {
		V3 c = v3(op.destination_box.center[0], op.destination_box.center[1], op.destination_box.center[2]);
		V3 q = pos_w - c;
		q = v3(q.x / op.scale[0], q.y / op.scale[1], q.z / op.scale[2]);
		V3 r = matTvec3(op.rotation, q);
		pos_w = (r + c) - v3(op.translation[0], op.translation[1], op.translation[2]);
		if (op.correct_dir) dir_w = warp_direction(matTvec3(op.rotation, unwarp_direction(dir_w)));
	} else if (op.hide_original && abox_contains(op.selection_box, pos_w)) {
		empty = true;
	}
}
void map_one(const NsbEditOp* ops, int n_ops, V3& pos_w, V3& dir_w, bool& empty) {
	for (int i = n_ops - 1; i >= 0; --i) { // reverse list order (testbed_nerf.cu:2899)
		if (ops[i].type == NSB_OP_CAGE) cage_map(ops[i], pos_w, dir_w, empty);
		else affine_map(ops[i], pos_w, dir_w, empty);
	}
}
// EditOperator::map_positions for one position, operators in reverse list order (testbed_nerf.cu:3595-3598): interpolate_tet_pos
// (cage_deformation.cu:136-192: no direction, and the vacated-region mask does not look at `copy`) and translate_in_box_pos
// (affine_duplication.cu:69-90: no direction)
void map_position_one(const NsbEditOp* ops, int n_ops, V3& pos_w, bool& empty) {
	for (int i = n_ops - 1; i >= 0; --i) {
		const NsbEditOp& op = ops[i];
		V3 d = v3(0.5f, 0.5f, 0.5f);
		if (op.type == NSB_OP_CAGE) {
			NsbEditOp pos_only = op;
			pos_only.copy = 0;
			pos_only.local_rotations = nullptr;
			cage_map(pos_only, pos_w, d, empty);
		} else {
			NsbEditOp pos_only = op;
			pos_only.correct_dir = 0;
			affine_map(pos_only, pos_w, d, empty);
		}
	}
}
// EditOperator::compute_poisson_residual_density for one position, operators in reverse list order (testbed_nerf.cu:3612-3620): the loop of
// compute_poisson_residual_density_kernel (cage_deformation.cu:341-383), h += (half) interpolated residual density, for the first tet of each
// operator that contains the (mapped, warped) position. Gated like CageDeformation::compute_poisson_residual_density (:647-672): only the
// residual density array has to be present. Returns how many operators added a residual; *last is the last one added.
int add_residual_density_one(const NsbEditOp* ops, int n_ops, V3 pos_w, uint16_t& h, uint16_t* last) {
	int n = 0;
	for (int k = n_ops - 1; k >= 0; --k) {
		const NsbEditOp& op = ops[k];
		if (op.type != NSB_OP_CAGE || !op.apply_poisson || op.n_tets == 0 || !op.boundary_residual_density) continue;
		Box saabb = mkbox(op.scene_aabb_min, op.scene_aabb_max);
		Box bbox = mkbox(op.bbox_min, op.bbox_max);
		V3 q = unwarp_position(pos_w, saabb);
		if (!box_contains(bbox, q)) continue;
		float b[4];
		int t = find_tet(op, q, b);
		if (t < 0) continue;
		const uint32_t* tv = op.tets + 4 * (size_t)t;
		float res = fmaf(b[3], op.boundary_residual_density[tv[3]], fmaf(b[2], op.boundary_residual_density[tv[2]],
		            fmaf(b[0], op.boundary_residual_density[tv[0]], b[1] * op.boundary_residual_density[tv[1]])));
		uint16_t r = f2h(res);
		if (last) *last = r;
		++n;
		h = hadd(h, r);                                                                              // half += half (:379)
	}
	return n;
}
// CageDeformation::compute_poisson_full_residuals gates on all three membrane arrays (cage_deformation.cu:675-716)
inline bool has_full_membrane(const NsbEditOp& op) {
	return op.type == NSB_OP_CAGE && op.apply_poisson && op.n_tets != 0 && op.boundary_shs && op.boundary_outside_density && op.boundary_residual_density;
}
// compute_residual_poisson_kernel (cage_deformation.cu:431-541) for one sample; outputs pre-zeroed by the caller.
void poisson_one(const NsbEditOp* ops, int n_ops, V3 pos_w, float* sh27, float* out_density, float* residual_density) {
	for (int i = n_ops - 1; i >= 0; --i) { // testbed_nerf.cu:2868
		const NsbEditOp& op = ops[i];
		if (!has_full_membrane(op)) continue;
		Box aabb = mkbox(op.scene_aabb_min, op.scene_aabb_max);
		Box bbox = mkbox(op.bbox_min, op.bbox_max);
		V3 p = unwarp_position(pos_w, aabb);
		if (!box_contains(bbox, p)) continue;
		float b[4];
		int t = find_tet(op, p, b);
		if (t < 0) continue;
		const uint32_t* tv = op.tets + 4 * (size_t)t;
		for (int k = 0; k < 27; ++k) {
			sh27[k] = fmaf(b[3], op.boundary_shs[27 * (size_t)tv[3] + k], fmaf(b[2], op.boundary_shs[27 * (size_t)tv[2] + k],
			          fmaf(b[0], op.boundary_shs[27 * (size_t)tv[0] + k], b[1] * op.boundary_shs[27 * (size_t)tv[1] + k])));
		}
		float od = fmaf(b[3], op.boundary_outside_density[tv[3]], fmaf(b[2], op.boundary_outside_density[tv[2]],
		           fmaf(b[0], op.boundary_outside_density[tv[0]], b[1] * op.boundary_outside_density[tv[1]])));
		float rd = fmaf(b[3], op.boundary_residual_density[tv[3]], fmaf(b[2], op.boundary_residual_density[tv[2]],
		           fmaf(b[0], op.boundary_residual_density[tv[0]], b[1] * op.boundary_residual_density[tv[1]])));
		*out_density = op.residual_amplitude * od;
		*residual_density = op.residual_amplitude * rd;
	}
}

// ----------------------------------------------------------------------------------------
// ray generation — init_rays_with_payload_kernel_nerf (testbed_nerf.cu:2512-2616),
// pixel_to_ray (common_device.cuh:245-295), advance_pos_nerf (:557-606)
// ----------------------------------------------------------------------------------------
struct Ray { V3 o, d; float t; bool alive; };

// ---- the general camera (ABI 3): pixel_to_ray with lens distortion, distortion map, depth of field (common_device.cuh:79-110,145-295),
// ld_random_val_2d / square2disk_shirley (random_val.cuh:109-127,278-282), read_envmap (envmap.cuh:30-62). Held to the frame tolerance, not bit-pinned.
static void apply_camera_distortion(const float* p, float u, float v, float& du, float& dv) {  // :145-160
	const float k1 = p[0], k2 = p[1], p1 = p[2], p2 = p[3];
	const float u2 = u * u, uv = u * v, v2 = v * v, r2 = u2 + v2;
	const float radial = k1 * r2 + k2 * r2 * r2;
	du = u * radial + 2.0f * p1 * uv + p2 * (r2 + 2.0f * u2);
	dv = v * radial + 2.0f * p2 * uv + p1 * (r2 + 2.0f * v2);
}
static void iterative_camera_undistortion(const float* params, float& u, float& v) {  // :163-197
	const float x0 = u, y0 = v;
	float x = u, y = v;
	for (uint32_t i = 0; i < 100u; ++i) {
		const float step0 = fmaxf(1.1920928955078125e-7f, fabsf(1e-6f * x));
		const float step1 = fmaxf(1.1920928955078125e-7f, fabsf(1e-6f * y));
		float dx, dy, dx0b, dy0b, dx0f, dy0f, dx1b, dy1b, dx1f, dy1f;
		apply_camera_distortion(params, x, y, dx, dy);
		apply_camera_distortion(params, x - step0, y, dx0b, dy0b);
		apply_camera_distortion(params, x + step0, y, dx0f, dy0f);
		apply_camera_distortion(params, x, y - step1, dx1b, dy1b);
		apply_camera_distortion(params, x, y + step1, dx1f, dy1f);
		const float j00 = 1.0f + (dx0f - dx0b) / (2.0f * step0), j01 = (dx1f - dx1b) / (2.0f * step1);
		const float j10 = (dy0f - dy0b) / (2.0f * step0), j11 = 1.0f + (dy1f - dy1b) / (2.0f * step1);
		const float rx = x + dx - x0, ry = y + dy - y0;
		const float invdet = 1.0f / (j00 * j11 - j10 * j01);  // Eigen's 2x2 inverse: adjugate times 1/det
		const float sx = (j11 * invdet) * rx + (-j01 * invdet) * ry;
		const float sy = (-j10 * invdet) * rx + (j00 * invdet) * ry;
		x -= sx; y -= sy;
		if (sx * sx + sy * sy < 1e-10f) break;
	}
	u = x; v = y;
}
static const uint32_t kSobolDir1[32] = {
	0x80000000u, 0xc0000000u, 0xa0000000u, 0xf0000000u, 0x88000000u, 0xcc000000u, 0xaa000000u, 0xff000000u, 0x80800000u, 0xc0c00000u, 0xa0a00000u,
	0xf0f00000u, 0x88880000u, 0xcccc0000u, 0xaaaa0000u, 0xffff0000u, 0x80008000u, 0xc000c000u, 0xa000a000u, 0xf000f000u, 0x88008800u, 0xcc00cc00u,
	0xaa00aa00u, 0xff00ff00u, 0x80808080u, 0xc0c0c0c0u, 0xa0a0a0a0u, 0xf0f0f0f0u, 0x88888888u, 0xccccccccu, 0xaaaaaaaau, 0xffffffffu,
};
static void ld_random_val_2d_general(uint32_t index, uint32_t seed, float& x, float& y) {
	index = nested_uniform_scramble_base2(index, seed);
	uint32_t X1 = 0;
	for (uint32_t bit = 0; bit < 32; ++bit) X1 ^= ((index >> bit) & 1u) * kSobolDir1[bit];
	x = (float)nested_uniform_scramble_base2(reverse_bits(index), hash_combine(seed, 0)) * 2.3283064365386963e-10f;
	y = (float)nested_uniform_scramble_base2(X1, hash_combine(seed, 1)) * 2.3283064365386963e-10f;
}
static void read_image2(const float* data, int rw, int rh, float px, float py, float& ox, float& oy) {  // read_image<2> :79-110
	const float fx = px * (float)(rw - 1), fy = py * (float)(rh - 1);
	const int tx = (int)fx, ty = (int)fy;
	const float wx = fx - (float)tx, wy = fy - (float)ty;
	auto rd = [&](int x, int y, int c) { x = std::max(std::min(x, rw - 1), 0); y = std::max(std::min(y, rh - 1), 0); return data[2 * ((size_t)x + (size_t)y * rw) + c]; };
	ox = (1.0f - wx) * (1.0f - wy) * rd(tx, ty, 0) + wx * (1.0f - wy) * rd(tx + 1, ty, 0) + (1.0f - wx) * wy * rd(tx, ty + 1, 0) + wx * wy * rd(tx + 1, ty + 1, 0);
	oy = (1.0f - wx) * (1.0f - wy) * rd(tx, ty, 1) + wx * (1.0f - wy) * rd(tx + 1, ty, 1) + (1.0f - wx) * wy * rd(tx, ty + 1, 1) + wx * wy * rd(tx + 1, ty + 1, 1);
}
static void read_envmap(const float* data, int rw, int rh, V3 dir, float* out4) {  // envmap.cuh:30-62 over dir_to_spherical_unorm (random_val.cuh:64-69)
	const float cos_theta = fminf(fmaxf(dir.y, -1.0f), 1.0f);
	const float theta = acosf(cos_theta);
	const float phi = atan2f(-dir.x, dir.z);
	const float cyl_x = theta / 3.14159265358979323846f, cyl_y = phi / (2.0f * 3.14159265358979323846f) + 0.5f;
	const float ex = cyl_y * (float)(rw - 1), ey = cyl_x * (float)(rh - 1);
	const int tx = (int)ex, ty = (int)ey;
	const float wx = ex - (float)tx, wy = ey - (float)ty;
	auto rd = [&](int x, int y) {
		if (x < 0) x += rw; else if (x >= rw) x -= rw;
		y = std::max(std::min(y, rh - 1), 0);
		return data + 4 * ((size_t)x + (size_t)y * rw);
	};
	const float *a = rd(tx, ty), *b = rd(tx + 1, ty), *c = rd(tx, ty + 1), *d = rd(tx + 1, ty + 1);
	const float w00 = (1.0f - wx) * (1.0f - wy), w10 = wx * (1.0f - wy), w01 = (1.0f - wx) * wy, w11 = wx * wy;
	for (int k = 0; k < 4; ++k) out4[k] = w00 * a[k] + w10 * b[k] + w01 * c[k] + w11 * d[k];
}
static bool general_camera(const NsbFrame& f) { return f.camera_distortion_mode != 0 || f.distortion_dev != nullptr || f.dof != 0.0f; }

Ray make_ray_general(const NsbFrame& f, uint32_t px, uint32_t py) {
	Ray r;
	r.alive = false;
	const uint32_t W = (uint32_t)f.width, H = (uint32_t)f.height, idx = px + W * py;
	const float fw = (float)W, fh = (float)H;
	const float u = ((float)px + 0.5f) * (1.0f / fw), v = ((float)py + 0.5f) * (1.0f / fh);
	const float rt = f.rolling_shutter[0] + f.rolling_shutter[1] * u + f.rolling_shutter[2] * v + f.rolling_shutter[3] * ld_random_val(f.spp_index, idx * 72239731u);
	float cam[12];
	for (int i = 0; i < 12; ++i) cam[i] = f.camera0[i] * rt + f.camera1[i] * (1.0f - rt);
	float off[2];
	ld_random_pixel_offset(f.snap_to_pixel_centers ? 0u : f.spp_index, off);
	const float uvx = ((float)px + off[0]) / fw, uvy = ((float)py + off[1]) / fh;
	const float* cd = f.camera_distortion_params;
	V3 dl;
	if (f.camera_distortion_mode == 2) {  // f_theta_undistortion (:232-245)
		const float xpix = (uvx - f.screen_center[0]) * cd[5], ypix = (uvy - f.screen_center[1]) * cd[6];
		const float norm = sqrtf(xpix * xpix + ypix * ypix);
		const float alpha = cd[0] + norm * (cd[1] + norm * (cd[2] + norm * (cd[3] + norm * cd[4])));
		float sa = sinf(alpha), ca = cosf(alpha);
		if (ca <= 1.17549435e-38f || norm == 0.0f) { r.o = v3(1000.0f, 0.0f, 0.0f); r.d = v3(0.0f, 0.0f, 1.0f); return r; }
		sa *= 1.0f / norm;
		dl = v3(sa * xpix, sa * ypix, ca);
	} else {
		dl = v3((uvx - f.screen_center[0]) * fw / f.focal_length[0], (uvy - f.screen_center[1]) * fh / f.focal_length[1], 1.0f);
		if (f.camera_distortion_mode == 1) iterative_camera_undistortion(cd, dl.x, dl.y);
	}
	if (f.distortion_dev) {
		float ox, oy;
		read_image2(f.distortion_dev, f.distortion_resolution[0], f.distortion_resolution[1], uvx, uvy, ox, oy);
		dl.x += ox; dl.y += oy;
	}
	V3 d = matvec3(cam, dl);
	V3 o = v3(cam[9], cam[10], cam[11]);
	if (f.dof != 0.0f) {
		const V3 lookat = v3(o.x + d.x * f.focus_z, o.y + d.y * f.focus_z, o.z + d.z * f.focus_z);
		float sx, sy;
		ld_random_val_2d_general(f.spp_index, px * 19349663u + py * 96925573u, sx, sy);
		const float a = sx * 2.0f - 1.0f, b = sy * 2.0f - 1.0f;  // square2disk_shirley
		float rr, phi;
		if (a * a > b * b) { rr = a; phi = (3.14159265358979323846f / 4.0f) * (b / a); }
		else { rr = b; phi = (3.14159265358979323846f / 2.0f) - (3.14159265358979323846f / 4.0f) * (a / b); }
		const float sp = sinf(phi), cp = cosf(phi);
		const float bx = f.dof * (rr * cp), by = f.dof * (rr * sp);
		o = v3(o.x + (cam[0] * bx + cam[3] * by), o.y + (cam[1] * bx + cam[4] * by), o.z + (cam[2] * bx + cam[5] * by));
		d = v3((lookat.x - o.x) / f.focus_z, (lookat.y - o.y) / f.focus_z, (lookat.z - o.z) / f.focus_z);
	}
	const float n2 = d.x * d.x + d.y * d.y + d.z * d.z;
	if (n2 > 0.0f) { const float n = sqrtf(n2); d = v3(d.x / n, d.y / n, d.z / n); }
	r.o = o;
	r.d = d;
	Box aabb = mkbox(f.render_aabb_min, f.render_aabb_max);
	float t = fmaxf(box_ray_tmin(aabb, r.o, r.d), NEAR_DISTANCE) + 1e-6f;
	if (!box_contains(aabb, madd3(r.d, t, r.o))) return r;
	r.t = t;
	r.alive = true;
	return r;
}

// glow_mode of composite_kernel_nerf (:807-903); returns the weight mask (mask_to_alpha)
static float glow_apply(int glow_mode, float glow_y_cutoff, V3 pos, V3 cam_origin, float* rgb) {
	float weight_mask = 1.0f, glow = 0.0f;
	const bool green_grid = glow_mode & 1, green_cutline = glow_mode & 2, mask_to_alpha = glow_mode & 4, radial_mode = glow_mode & 8, grid_mode = glow_mode & 16;
	float dist;
	if (radial_mode) {
		const V3 q = pos - cam_origin;
		dist = sqrtf(q.x * q.x + q.y * q.y + q.z * q.z);
		dist = fminf(dist, (4.5f - pos.y) * 0.333f);
	} else {
		dist = pos.y;
	}
	if (grid_mode) {
		glow = 1.0f / fmaxf(1.0f, dist);
	} else {
		float y = glow_y_cutoff - dist;
		float mask = 0.0f;
		if (y > 0.0f) {
			y *= 80.0f;
			mask = fminf(1.0f, y);
			if (green_cutline) glow += fmaxf(0.0f, 1.0f - fabsf(1.0f - y)) * 4.0f;
			if (y > 1.0f) y = 1.0f - (y - 1.0f) * 0.05f;
			if (green_grid) glow += fmaxf(0.0f, y / fmaxf(1.0f, dist));
		}
		if (mask_to_alpha) weight_mask = mask;
	}
	if (glow > 0.0f) {
		float line = 0.0f;
		const float pi = 3.141592653589793f;
		for (int k = 0; k < 4; ++k) {
			const float m = (float)(2 << k);
			line += fmaxf(0.0f, cosf(pos.y * m * pi * 16.0f) - 0.975f);
			line += fmaxf(0.0f, cosf(pos.x * m * pi * 16.0f) - 0.975f);
			line += fmaxf(0.0f, cosf(pos.z * m * pi * 16.0f) - 0.975f);
		}
		if (grid_mode) {
			glow = glow * line * 15.0f;
			rgb[1] = glow; rgb[2] = glow * 0.5f; rgb[0] = glow * 0.25f;
		} else {
			glow = glow * glow * 0.25f + glow * line * 15.0f;
			rgb[1] += glow; rgb[2] += glow * 0.5f; rgb[0] += glow * 0.25f;
		}
	}
	return weight_mask;
}

Ray make_ray(const NsbFrame& f, uint32_t px, uint32_t py) {
	if (general_camera(f)) return make_ray_general(f, px, py);
	Ray r;
	r.alive = false;
	uint32_t W = (uint32_t)f.width, H = (uint32_t)f.height;
	uint32_t idx = px + W * py;
	float u = ((float)px + 0.5f) * (1.0f / (float)W);
	float v = ((float)py + 0.5f) * (1.0f / (float)H);
	float rt = f.rolling_shutter[0];
	rt = fmaf(f.rolling_shutter[1], u, rt);
	rt = fmaf(f.rolling_shutter[2], v, rt);
	rt = fmaf(f.rolling_shutter[3], ld_random_val(f.spp_index, idx * 72239731u), rt);
	float cam[12];
	for (int i = 0; i < 12; ++i) cam[i] = fmaf(f.camera0[i], rt, f.camera1[i] * (1.0f - rt));
	float off[2];
	ld_random_pixel_offset(f.snap_to_pixel_centers ? 0u : f.spp_index, off);
	float uvx = ((float)px + off[0]) / (float)W;
	float uvy = ((float)py + off[1]) / (float)H;
	V3 dl = v3((uvx - f.screen_center[0]) * (float)W / f.focal_length[0], (uvy - f.screen_center[1]) * (float)H / f.focal_length[1], 1.0f);
	V3 d = matvec3(cam, dl);
	r.o = v3(cam[9], cam[10], cam[11]);
	float n2 = dot3(d, d);
	if (n2 > 0.0f) { float n = sqrtf(n2); d = v3(d.x / n, d.y / n, d.z / n); } // Eigen normalized()
	r.d = d;
	Box aabb = mkbox(f.render_aabb_min, f.render_aabb_max);
	float t = fmaxf(box_ray_tmin(aabb, r.o, r.d), NEAR_DISTANCE) + 1e-6f;
	if (!box_contains(aabb, madd3(r.d, t, r.o))) return r;
	r.t = t;
	r.alive = true;
	return r;
}

// Finds the next occupied sample position at or after r.t (inner loop of advance_pos_nerf :588-603 and
// generate_next_nerf_network_inputs :671-688). Returns false when the ray leaves the render AABB.
bool next_occupied(const NsbFrame& f, const uint8_t* bitfield, const Ray& r, V3 idir, float& t, float& dt, V3& pos, uint32_t& mip_out, uint32_t& cell_out) {
	Box aabb = mkbox(f.render_aabb_min, f.render_aabb_max);
	float cone = f.cone_angle_constant;
	while (true) {
		pos = madd3(r.d, t, r.o);
		if (!box_contains(aabb, pos)) return false;
		dt = calc_dt(t, cone);
		uint32_t mip = (uint32_t)std::max(f.min_mip, mip_from_dt(dt, pos));
		uint32_t cell = cascaded_grid_idx_at(pos, mip);
		if (!bitfield || bitfield_at(cell, mip, bitfield)) { mip_out = mip; cell_out = cell; return true; }
		uint32_t res = GRIDSIZE >> mip;
		t = advance_to_next_voxel(t, cone, pos, r.d, idir, res);
	}
}

struct Scene {
	Model model;
	const uint8_t* bitfield;
	const NsbEditOp* ops;
	int n_ops;
};

} // namespace

// ========================================================================================
// C entry points (ctypes)
// ========================================================================================
// ---- tcnn::default_rng_t = pcg32 (PCG-XSH-RR 64/32; public algorithm, tiny-cuda-nn pcg32.h [tcnn-ext]) -------------------
// Pinned by the PCG reference known-answer vector (seed 42, stream 54) in tests/test_oracle_units.py.
struct Pcg32 {
	uint64_t state, inc;
	uint32_t next_uint() {
		uint64_t old = state;
		state = old * 0x5851f42d4c957f2dULL + inc;
		uint32_t xorshifted = (uint32_t)(((old >> 18u) ^ old) >> 27u);
		uint32_t rot = (uint32_t)(old >> 59u);
		return (xorshifted >> rot) | (xorshifted << ((~rot + 1u) & 31u));
	}
	float next_float() {
		uint32_t u = (next_uint() >> 9) | 0x3f800000u;
		float f;
		memcpy(&f, &u, 4);
		return f - 1.0f;
	}
	void seed(uint64_t initstate, uint64_t initseq) {
		state = 0u;
		inc = (initseq << 1u) | 1u;
		next_uint();
		state += initstate;
		next_uint();
	}
	void advance(uint64_t delta) {
		uint64_t cur_mult = 0x5851f42d4c957f2dULL, cur_plus = inc, acc_mult = 1u, acc_plus = 0u;
		while (delta > 0) {
			if (delta & 1) { acc_mult *= cur_mult; acc_plus = acc_plus * cur_mult + cur_plus; }
			cur_plus = (cur_mult + 1) * cur_plus;
			cur_mult *= cur_mult;
			delta >>= 1;
		}
		state = acc_mult * state + acc_plus;
	}
};

extern "C" {

typedef struct {
	NsbModelDesc desc;
	const uint16_t* params;
	uint64_t n_params;
	const uint8_t* bitfield; // may be NULL (no occupancy grid)
	const NsbEditOp* ops;
	int32_t n_ops;
} OrcScene;

typedef struct {
	uint64_t n_rays, n_rays_alive, n_hit, n_samples, n_old_samples;
	int32_t threads;
} OrcStats;

int orc_model_n_params(const NsbModelDesc* d, uint64_t* n) {
	Model m;
	if (!model_init(m, d, nullptr, 0)) return 1;
	*n = m.n_params;
	return 0;
}
// level table (scale, res, offset, size) x n_levels, for tests of the encoding geometry
int orc_level_table(const NsbModelDesc* d, float* scale, uint32_t* res, uint32_t* offset, uint32_t* size) {
	Model m;
	if (!model_init(m, d, nullptr, 0)) return 1;
	for (uint32_t l = 0; l < d->n_levels; ++l) { scale[l] = m.levels[l].scale; res[l] = m.levels[l].res; offset[l] = m.levels[l].offset; size[l] = m.levels[l].size; }
	return 0;
}

// tcnn's grid_index on one level for n grid coordinates g (n x 3): the uint32 index into the level; 1 for a rejected description or level
int orc_grid_index(const NsbModelDesc* d, uint32_t level, const uint32_t* g, uint32_t n, uint32_t* out) {
	Model m;
	if (!model_init(m, d, nullptr, 0) || level >= d->n_levels) return 1;
	for (uint32_t i = 0; i < n; ++i) out[i] = grid_entry(m.levels[level], g + 3 * (size_t)i);
	return 0;
}
int32_t orc_f2i(float v) { return cvt_rzi_s32(v); }

uint16_t orc_f2h(float f) { return f2h(f); }
float orc_h2f(uint16_t h) { return h2f(h); }
float orc_ld_random_val(uint32_t index, uint32_t seed) { return ld_random_val(index, seed); }
void orc_pixel_offset(uint32_t spp, float* off) { ld_random_pixel_offset(spp, off); }
uint32_t orc_morton3D(uint32_t x, uint32_t y, uint32_t z) { return morton3D(x, y, z); }
int orc_mip_from_pos(float x, float y, float z) { return mip_from_pos(v3(x, y, z)); }
uint32_t orc_cascaded_grid_idx_at(float x, float y, float z, uint32_t mip) { return cascaded_grid_idx_at(v3(x, y, z), mip); }

// coords: n x 7 floats (NerfCoordinate). out: fp16 row-major [rows x n].
int orc_encode(const OrcScene* s, const float* coords, uint32_t n, uint16_t* out /*32 x n*/) {
	Model m;
	if (!model_init(m, &s->desc, s->params, s->n_params)) return 1;
#pragma omp parallel for schedule(static)
	for (int64_t i = 0; i < (int64_t)n; ++i) {
		uint16_t f[32];
		encode_grid(m, v3(coords[7 * i], coords[7 * i + 1], coords[7 * i + 2]), f);
		for (int k = 0; k < 32; ++k) out[(size_t)k * n + i] = f[k];
	}
	return 0;
}
int orc_inference(const OrcScene* s, const float* coords, uint32_t n, uint16_t* out /*16 x n*/, int density_only) {
	Model m;
	if (!model_init(m, &s->desc, s->params, s->n_params)) return 1;
#pragma omp parallel for schedule(static)
	for (int64_t i = 0; i < (int64_t)n; ++i) {
		uint16_t o[16], d[16];
		network_forward(m, v3(coords[7 * i], coords[7 * i + 1], coords[7 * i + 2]), v3(coords[7 * i + 4], coords[7 * i + 5], coords[7 * i + 6]), o, d, density_only != 0);
		const uint16_t* src = density_only ? d : o;
		for (int k = 0; k < 16; ++k) out[(size_t)k * n + i] = src[k];
	}
	return 0;
}
int orc_map_rays(const OrcScene* s, float* coords, uint8_t* empty_mask, uint32_t n) {
#pragma omp parallel for schedule(static)
	for (int64_t i = 0; i < (int64_t)n; ++i) {
		V3 p = v3(coords[7 * i], coords[7 * i + 1], coords[7 * i + 2]);
		V3 d = v3(coords[7 * i + 4], coords[7 * i + 5], coords[7 * i + 6]);
		bool empty = false;
		map_one(s->ops, s->n_ops, p, d, empty);
		coords[7 * i] = p.x; coords[7 * i + 1] = p.y; coords[7 * i + 2] = p.z;
		coords[7 * i + 4] = d.x; coords[7 * i + 5] = d.y; coords[7 * i + 6] = d.z;
		empty_mask[i] = empty ? 1 : 0;
	}
	return 0;
}
int orc_poisson_residuals(const OrcScene* s, const float* coords, uint32_t n, float* sh, float* out_density, float* residual_density) {
#pragma omp parallel for schedule(static)
	for (int64_t i = 0; i < (int64_t)n; ++i) {
		for (int k = 0; k < 27; ++k) sh[27 * i + k] = 0.0f;
		out_density[i] = 0.0f;
		residual_density[i] = 0.0f;
		poisson_one(s->ops, s->n_ops, v3(coords[7 * i], coords[7 * i + 1], coords[7 * i + 2]), sh + 27 * i, out_density + i, residual_density + i);
	}
	return 0;
}
// EditOperator::map_positions over all operators: positions (warped) are `stride` floats apart, mapped in place; the mask (optional) is only
// ever set, like nsb_map_positions for one operator.
int orc_map_positions(const OrcScene* s, float* positions, uint32_t stride, uint8_t* empty_mask, uint32_t n) {
	if (stride < 3) return 1;
#pragma omp parallel for schedule(static)
	for (int64_t i = 0; i < (int64_t)n; ++i) {
		float* q = positions + (size_t)i * stride;
		V3 p = v3(q[0], q[1], q[2]);
		bool empty = false;
		map_position_one(s->ops, s->n_ops, p, empty);
		q[0] = p.x; q[1] = p.y; q[2] = p.z;
		if (empty && empty_mask) empty_mask[i] = 1;
	}
	return 0;
}
// EditOperator::compute_poisson_residual_density over all operators: density_fp16[i] += each operator's residual density at position i
int orc_poisson_residual_density(const OrcScene* s, const float* positions, uint32_t stride, uint16_t* density_fp16, uint32_t n) {
	if (stride < 3) return 1;
#pragma omp parallel for schedule(static)
	for (int64_t i = 0; i < (int64_t)n; ++i) {
		const float* q = positions + (size_t)i * stride;
		add_residual_density_one(s->ops, s->n_ops, v3(q[0], q[1], q[2]), density_fp16[i], nullptr);
	}
	return 0;
}

// Occupancy march without termination. rec: n_pixels*max_samples*5 floats (t, dt, x, y, z);
// idx: n_pixels*max_samples*2 (mip, cell); count: total occupied samples on the ray.
int orc_march_trace(const OrcScene* s, const NsbFrame* f, const uint32_t* pixels, uint32_t n_pixels, uint32_t max_samples,
                    float* rec, uint32_t* idx, uint32_t* count) {
#pragma omp parallel for schedule(dynamic, 16)
	for (int64_t i = 0; i < (int64_t)n_pixels; ++i) {
		uint32_t pix = pixels[i];
		uint32_t px = pix % (uint32_t)f->width, py = pix / (uint32_t)f->width;
		Ray r = make_ray(*f, px, py);
		uint32_t c = 0;
		if (r.alive) {
			V3 idir = v3(1.0f / r.d.x, 1.0f / r.d.y, 1.0f / r.d.z);
			float t = r.t;
			float dt0 = calc_dt(t, f->cone_angle_constant);
			t = fmaf(ld_random_val(f->spp_index, pix * 786433u), dt0, t);
			while (c < MARCH_ITER) {
				float dt; V3 pos; uint32_t mip, cell;
				if (!next_occupied(*f, s->bitfield, r, idir, t, dt, pos, mip, cell)) break;
				if (c < max_samples) {
					float* rr = rec + ((size_t)i * max_samples + c) * 5;
					rr[0] = t; rr[1] = dt; rr[2] = pos.x; rr[3] = pos.y; rr[4] = pos.z;
					uint32_t* ii = idx + ((size_t)i * max_samples + c) * 2;
					ii[0] = mip; ii[1] = cell;
				}
				++c;
				t += dt;
			}
		}
		count[i] = c;
	}
	return 0;
}

// Full frame: Testbed::render_nerf with the trace loop restated per ray (the per-ray result of the
// reference does not depend on how rays are batched into rounds: every GEMM column is independent and
// composite_kernel_nerf :750-955 walks a ray's samples strictly in order).
// fb: float4[W*H] in/out (over-blended like shade_kernel_nerf :2479), depth: float[W*H] out.
// margin (optional, float[W*H]): min over a ray's steps of |A - (1 - min_transmittance)| — pixels whose
// margin is below float noise can legitimately flip the early-termination branch on other hardware.
int orc_render(const OrcScene* s, const NsbFrame* f, float* fb, float* depth, OrcStats* stats, float* margin) {
	Model m;
	if (!model_init(m, &s->desc, s->params, s->n_params)) return 1;
	const int W = f->width, H = f->height;
	const Box train = mkbox(f->train_aabb_min, f->train_aabb_max);
	const bool ops_on = f->apply_operators && s->n_ops > 0;
	bool any_poisson = false;
	if (ops_on) for (int i = 0; i < s->n_ops; ++i) any_poisson |= has_full_membrane(s->ops[i]);
	uint64_t n_alive = 0, n_hit = 0, n_samples = 0, n_old = 0;
	const V3 cam_fwd = v3(f->camera1[6], f->camera1[7], f->camera1[8]);
	const V3 cam_org = v3(f->camera1[9], f->camera1[10], f->camera1[11]);
#pragma omp parallel for schedule(dynamic, 1) reduction(+ : n_alive, n_hit, n_samples, n_old)
	for (int py = 0; py < H; ++py) {
		for (int px = 0; px < W; ++px) {
			uint32_t pix = (uint32_t)px + (uint32_t)W * (uint32_t)py;
			depth[pix] = 1e10f; // :2581
			if (margin) margin[pix] = 1e30f;
			Ray r = make_ray(*f, (uint32_t)px, (uint32_t)py);
			if (f->envmap_dev) read_envmap(f->envmap_dev, f->envmap_resolution[0], f->envmap_resolution[1], r.d, fb + 4 * (size_t)pix);  // :2581-2583, every pixel
			if (!r.alive) continue;
			if (f->render_mode == NSB_RENDER_DISTORTION) {  // :2596-2607
				float dx = 0.5f, dy = 0.5f;
				if (f->distortion_dev) {
					read_image2(f->distortion_dev, f->distortion_resolution[0], f->distortion_resolution[1], ((float)px + 0.5f) / (float)W, ((float)py + 0.5f) / (float)H, dx, dy);
					dx = dx * 50.0f + 0.5f; dy = dy * 50.0f + 0.5f;
				}
				float* o4 = fb + 4 * (size_t)pix;
				o4[0] = dx; o4[1] = dy; o4[2] = 0.5f; o4[3] = 1.0f;
				depth[pix] = 1.0f;
				continue;
			}
			++n_alive;
			V3 idir = v3(1.0f / r.d.x, 1.0f / r.d.y, 1.0f / r.d.z);
			float t = r.t;
			t = fmaf(ld_random_val(f->spp_index, pix * 786433u), calc_dt(t, f->cone_angle_constant), t); // :585
			float rgba[4] = {0, 0, 0, 0};
			float local_depth = 0.0f, max_weight = 0.0f;
			uint32_t n_steps = 0;
			float mrg = 1e30f;
			bool done = false; // left the AABB or saturated; a ray still marching after MARCH_ITER steps is dropped (:2812)
			for (uint32_t step = 1; step < MARCH_ITER; ++step) {
				float dt; V3 pos; uint32_t mip, cell;
				// payload.n_steps = j + current_step (:959): samples composited, +1 when the ray ends by leaving the AABB
				if (!next_occupied(*f, s->bitfield, r, idir, t, dt, pos, mip, cell)) { done = true; ++n_steps; break; }
				// generate_next_nerf_network_inputs :690
				V3 pw = warp_position(pos, train);
				V3 dw = warp_direction(r.d);
				float dtw = warp_dt(dt);
				t += dt;
				++n_samples;
				++n_steps;
				// membrane residuals in deformed space (:2867-2883), then the backward map (:2896-2904)
				float sh27[27], dob = 0.0f, drb = 0.0f;
				bool empty = false;
				uint16_t out_old[16];
				bool have_old = false;
				if (ops_on) {
					if (any_poisson) {
						for (int k = 0; k < 27; ++k) sh27[k] = 0.0f;
						poisson_one(s->ops, s->n_ops, pw, sh27, &dob, &drb);
						if (dob > 1e-9f && f->poisson_target) { // only place the "old" inference is read (:773)
							uint16_t dummy[16];
							network_forward(m, pw, dw, dummy, out_old, true);
							have_old = true;
							++n_old;
						}
					}
					map_one(s->ops, s->n_ops, pw, dw, empty);
				}
				uint16_t out[16];
				network_forward(m, pw, dw, out, nullptr, false);
				// composite_kernel_nerf :750-955 (one sample)
				V3 cpos = unwarp_position(pw, train);
				float T = 1.0f - rgba[3];
				float dtu = unwarp_dt(dtw);
				float alpha;
				float sigma = network_to_density(h2f(out[3]), f->density_activation);
				if (empty) {
					alpha = 0.0f;
				} else if (dob > 1e-9f) {
					float val;
					if (f->poisson_target) {
						float target = network_to_density(h2f(have_old ? out_old[0] : (uint16_t)0), f->density_activation);
						val = fminf(fmaxf(target, sigma), sigma + drb);
					} else {
						val = sigma + drb;
					}
					alpha = 1.0f - expf(-val * dtu);
				} else {
					alpha = 1.0f - expf(-sigma * dtu);
				}
				if (f->show_accel) alpha = 1.0f;  // testbed_nerf.cu:788-790
				float weight = alpha * T;
				float rgb[3];
				for (int c = 0; c < 3; ++c) rgb[c] = network_to_rgb(h2f(out[c]), f->rgb_activation);
				if (f->glow_mode) {  // :807-903
					const float mask = glow_apply(f->glow_mode, f->glow_y_cutoff, cpos, cam_org, rgb);
					if (f->glow_mode & 4) weight *= mask;
				}
				if (f->render_mode == NSB_RENDER_AO) { rgb[0] = rgb[1] = rgb[2] = alpha; }
				else if (f->render_mode == NSB_RENDER_POSITIONS && f->show_accel) {  // :913-923: one random colour per occupancy cell
					uint32_t mip = (uint32_t)std::max(f->min_mip, mip_from_pos(cpos));
					float res = (float)(GRIDSIZE >> mip);
					int ix = (int)(cpos.x * res), iy = (int)(cpos.y * res), iz = (int)(cpos.z * res);
					Pcg32 rng;  // tcnn::default_rng_t rng(seed) = pcg32::seed(initstate, 1)
					rng.seed((uint64_t)(int64_t)(ix + iy * 232323 + iz * 727272), 1);
					rgb[0] = 1.0f - (float)mip * 0.25f;
					rgb[1] = rng.next_float();
					rgb[2] = rng.next_float();
				}
				else if (f->render_mode == NSB_RENDER_POSITIONS) { rgb[0] = (cpos.x - 0.5f) / 2.0f + 0.5f; rgb[1] = (cpos.y - 0.5f) / 2.0f + 0.5f; rgb[2] = (cpos.z - 0.5f) / 2.0f + 0.5f; }
				else if (f->render_mode == NSB_RENDER_DEPTH) { float z = dot3(cam_fwd, cpos - r.o) * f->depth_scale; rgb[0] = rgb[1] = rgb[2] = z; }
				else if (f->render_mode == NSB_RENDER_DISTANCE) { V3 q = cpos - r.o; float z = sqrtf(dot3(q, q)) * f->depth_scale; rgb[0] = rgb[1] = rgb[2] = z; }
				else if (f->render_mode == NSB_RENDER_STEPSIZE) { float wdt = warp_dt(dtu); rgb[0] = rgb[1] = rgb[2] = wdt; }
				if (dob > 1e-9f) {
					float alpha_N = 1.0f - expf(-sigma * dtu);
					float alpha_R = 1.0f - expf(-dob * dtu);
					float w_N = alpha_N / (alpha_N + alpha_R), w_R = alpha_R / (alpha_N + alpha_R);
					float res[3];
					evaluate_sh9(sh27, unwarp_direction(dw), res);
					for (int c = 0; c < 3; ++c) rgba[c] = fmaf(weight, fmaf(w_R, res[c], w_N * rgb[c]), rgba[c]);
				} else {
					for (int c = 0; c < 3; ++c) rgba[c] = fmaf(rgb[c], weight, rgba[c]);
				}
				rgba[3] += weight;
				if (weight > max_weight) { max_weight = weight; local_depth = dot3(cam_fwd, cpos - cam_org); }
				mrg = fminf(mrg, fabsf(rgba[3] - (1.0f - f->min_transmittance)));
				if (rgba[3] > (1.0f - f->min_transmittance)) {
					float a = rgba[3];
					for (int c = 0; c < 4; ++c) rgba[c] /= a;
					done = true;
					break;
				}
			}
			if (margin) margin[pix] = mrg;
			if (!done) continue;
			// compact_kernel_nerf :2503 + shade_kernel_nerf :2464-2482
			if (rgba[3] > 0.001f) {
				++n_hit;
				float tmp[4] = {rgba[0], rgba[1], rgba[2], rgba[3]};
				if (f->render_mode == NSB_RENDER_COST) { float col = (float)n_steps / 128.0f; tmp[0] = tmp[1] = tmp[2] = col; tmp[3] = 1.0f; }
				if (!f->linear_colors && f->render_mode == NSB_RENDER_SHADE) for (int c = 0; c < 3; ++c) tmp[c] = srgb_to_linear(tmp[c]);
				for (int c = 0; c < 4; ++c) fb[4 * (size_t)pix + c] = fmaf(fb[4 * (size_t)pix + c], (1.0f - tmp[3]), tmp[c]);
				if (tmp[3] > 0.2f) depth[pix] = local_depth;
			}
		}
	}
	if (stats) {
		stats->n_rays = (uint64_t)W * H;
		stats->n_rays_alive = n_alive;
		stats->n_hit = n_hit;
		stats->n_samples = n_samples;
		stats->n_old_samples = n_old;
#ifdef _OPENMP
		stats->threads = omp_get_max_threads();
#else
		stats->threads = 1;
#endif
	}
	return 0;
}

// accumulate_kernel (render_buffer.cu:217-258) and tonemap_kernel (:471-499, curves :262-332) on host buffers
static inline float linear_to_srgb_(float l) { return l < 0.0031308f ? 12.92f * l : 1.055f * powf(l, 0.41666f) - 0.055f; }
int orc_accumulate(const float* frame, float* acc, int n, float sample_count, int color_space) {
	for (int i = 0; i < n; ++i) {
		float c[4] = {frame[4 * i], frame[4 * i + 1], frame[4 * i + 2], frame[4 * i + 3]};
		float* t = acc + 4 * (size_t)i;
		const float inv = sample_count + 1.0f;
		if (color_space == NSB_COLOR_VISPOSNEG) {
			float val = c[0] - c[1], tv = t[0] - t[1];
			tv = (tv * sample_count + val) / inv;
			t[0] = fmaxf(tv, 0.0f); t[1] = fmaxf(-tv, 0.0f);
		} else {
			if (color_space == NSB_COLOR_SRGB) for (int k = 0; k < 3; ++k) c[k] = linear_to_srgb_(c[k]);
			for (int k = 0; k < 3; ++k) t[k] = (t[k] * sample_count + c[k]) / inv;
		}
		t[3] = (t[3] * sample_count + c[3]) / inv;
	}
	return 0;
}
int orc_tonemap(const float* acc, float* out, int n, const NsbTonemap* p) {
	for (int i = 0; i < n; ++i) {
		float bg[4] = {p->background_color[0], p->background_color[1], p->background_color[2], p->background_color[3]};
		if (p->color_space != NSB_COLOR_SRGB) for (int k = 0; k < 3; ++k) bg[k] = srgb_to_linear(bg[k]);
		float c[3] = {acc[4 * i], acc[4 * i + 1], acc[4 * i + 2]};
		float a = acc[4 * i + 3];
		float weight = (1.0f - a) * bg[3];
		for (int k = 0; k < 3; ++k) c[k] += bg[k] * weight;
		a += weight;
		if (p->color_space == NSB_COLOR_SRGB) for (int k = 0; k < 3; ++k) c[k] = srgb_to_linear(c[k]);
		const float e = powf(2.0f, p->exposure);
		for (int k = 0; k < 3; ++k) c[k] *= e;
		if (p->tonemap_curve != NSB_TONEMAP_IDENTITY) {
			for (int k = 0; k < 3; ++k) c[k] = fmaxf(c[k], 0.0f);
			if (p->tonemap_curve == NSB_TONEMAP_REINHARD) {
				float Y = 0.2126f * c[0] + (0.7152f * c[1] + 0.0722f * c[2]);  // luminance_coefficients.dot(x): Eigen's x0 + (x1 + x2)
				for (int k = 0; k < 3; ++k) c[k] *= 1.0f / (Y + 1.0f);
			} else {
				float k0, k1, k2, k3, k4, k5;
				if (p->tonemap_curve == NSB_TONEMAP_ACES) {
					k0 = 0.6f * 0.6f * 2.51f; k1 = 0.6f * 0.03f; k2 = 0.0f; k3 = 0.6f * 0.6f * 2.43f; k4 = 0.6f * 0.59f; k5 = 0.14f;
				} else {
					const float A = 0.15f, B = 0.50f, C = 0.10f, D = 0.20f, E = 0.02f, F = 0.30f;
					k0 = A * F - A * E; k1 = C * B * F - B * E; k2 = 0.0f; k3 = A * F; k4 = B * F; k5 = D * F * F;
					const float W = 11.2f;
					const float white_scale = (k3 * (W * W) + k4 * W + k5) / (k0 * (W * W) + k1 * W + k2);
					k0 = 4.0f * k0 * white_scale; k1 = 2.0f * k1 * white_scale; k2 = k2 * white_scale; k3 = 4.0f * k3; k4 = 2.0f * k4;
				}
				for (int k = 0; k < 3; ++k) { float sq = c[k] * c[k]; c[k] = (sq * k0 + k1 * c[k] + k2) / (k3 * sq + k4 * c[k] + k5); }
			}
		}
		if (p->output_color_space == NSB_COLOR_SRGB) for (int k = 0; k < 3; ++k) c[k] = linear_to_srgb_(c[k]);
		if (p->clamp_output_color) { for (int k = 0; k < 3; ++k) c[k] = fminf(fmaxf(c[k], 0.0f), 1.0f); a = fminf(fmaxf(a, 0.0f), 1.0f); }
		out[4 * i] = c[0]; out[4 * i + 1] = c[1]; out[4 * i + 2] = c[2]; out[4 * i + 3] = a;
	}
	return 0;
}

// update_density_grid_mean_and_bitfield (testbed_nerf.cu:3642-3658) + grid_to_bitfield (:514) + bitfield_max_pool (:534)
static inline uint32_t morton3D_invert_(uint32_t x) {
	x = x & 0x49249249u;
	x = (x | (x >> 2)) & 0xc30c30c3u;
	x = (x | (x >> 4)) & 0x0f00f00fu;
	x = (x | (x >> 8)) & 0xff0000ffu;
	x = (x | (x >> 16)) & 0x0000ffffu;
	return x;
}
int orc_density_grid_to_bitfield(const float* grid /*5*128^3*/, uint8_t* bits /*5*128^3/8*/, float* mean_out) {
	double sum = 0.0;
	for (uint32_t i = 0; i < GRIDVOL; ++i) sum += (double)fmaxf(grid[i], 0.0f);
	float mean = (float)(sum / (double)GRIDVOL);
	float thresh = std::min(0.01f, mean);
	for (uint32_t i = 0; i < GRIDVOL / 8 * (uint32_t)CASCADES; ++i) {
		uint8_t b = 0;
		for (int j = 0; j < 8; ++j) b |= grid[(size_t)i * 8 + j] > thresh ? (uint8_t)(1u << j) : (uint8_t)0;
		bits[i] = b;
	}
	for (int level = 1; level < CASCADES; ++level) {
		const uint8_t* prev = bits + (size_t)(level - 1) * (GRIDVOL / 8);
		uint8_t* next = bits + (size_t)level * (GRIDVOL / 8);
		for (uint32_t i = 0; i < GRIDVOL / 64; ++i) {
			uint8_t b = 0;
			for (int j = 0; j < 8; ++j) b |= prev[(size_t)i * 8 + j] > 0 ? (uint8_t)(1u << j) : (uint8_t)0;
			uint32_t x = morton3D_invert_(i >> 0) + GRIDSIZE / 8, y = morton3D_invert_(i >> 1) + GRIDSIZE / 8, z = morton3D_invert_(i >> 2) + GRIDSIZE / 8;
			next[morton3D(x, y, z)] |= b;
		}
	}
	if (mean_out) *mean_out = mean;
	return 0;
}

void orc_pcg32_seed(uint64_t initstate, uint64_t initseq, uint64_t* state_inc /*2*/) {
	Pcg32 r; r.seed(initstate, initseq);
	state_inc[0] = r.state; state_inc[1] = r.inc;
}
void orc_pcg32_next(uint64_t* state_inc, uint32_t n, uint32_t* out) {
	Pcg32 r{state_inc[0], state_inc[1]};
	for (uint32_t i = 0; i < n; ++i) out[i] = r.next_uint();
	state_inc[0] = r.state;
}
void orc_pcg32_advance(uint64_t* state_inc, uint64_t delta) {
	Pcg32 r{state_inc[0], state_inc[1]};
	r.advance(delta);
	state_inc[0] = r.state;
}

// Testbed::update_density_grid_nerf_operator (testbed_nerf.cu:3533-3639) on the host; `grid` is the running density grid
// (in/out, 5*128^3), `bits` receives update_density_grid_mean_and_bitfield's result. `samples_out` (optional, n x 4 floats)
// receives {mapped warped position, activated+residual density} per sample for diagnostics. `cells_out` (optional, n uint32) receives
// each sample's splat cell (cascade * 128^3 + Morton index) and `residual_out` (optional, n fp16 bits) the membrane residual half
// added to its activated density: 0 if none was added, NaN (0x7e00) if more than one operator added one.
int orc_update_density_grid(const OrcScene* s, const NsbGridUpdate* u, float* grid, uint8_t* bits, float* mean_out, float* samples_out,
                            uint32_t* cells_out, uint16_t* residual_out) {
	Model m;
	if (!model_init(m, &s->desc, s->params, s->n_params)) return 1;
	const uint32_t n_cells = GRIDVOL * (uint32_t)CASCADES;
	if (u->reset_grid) memset(grid, 0, (size_t)n_cells * 4);                                   // :3558-3560
	std::vector<uint32_t> tmp(n_cells, 0u);                                                    // density_grid_tmp, as uint bits (:3563)
	const uint32_t n_total = u->n_uniform_samples + u->n_nonuniform_samples;
	const Box aabb = mkbox(u->train_aabb_min, u->train_aabb_max);
	const uint32_t n_cascades = (uint32_t)u->n_cascades;
#pragma omp parallel for schedule(dynamic, 1024)
	for (int64_t ii = 0; ii < (int64_t)n_total; ++ii) {
		const uint32_t i = (uint32_t)ii;
		// generate_grid_samples_nerf_nonuniform (common_nerf.cu:179-208): two launches, m_rng.advance() (2^32) after the first
		const bool second = i >= u->n_uniform_samples;
		const uint32_t li = second ? i - u->n_uniform_samples : i;
		const uint32_t n_el = second ? u->n_nonuniform_samples : u->n_uniform_samples;
		const float thresh = second ? 0.01f : -0.01f;
		Pcg32 rng{u->rng_state, u->rng_inc};
		if (second) rng.advance(1ull << 32);
		rng.advance((uint64_t)(li * 4u));
		const uint32_t level = (uint32_t)(rng.next_float() * (float)n_cascades) % n_cascades;
		uint32_t idx = 0;
		for (uint32_t j = 0; j < 10; ++j) {
			idx = ((li + u->ema_step * n_el) * 56924617u + j * 19349663u + 96925573u) % GRIDVOL;
			idx += level * GRIDVOL;
			if (grid[idx] > thresh) break;
		}
		const uint32_t pos_idx = idx % GRIDVOL;
		const float x = (float)morton3D_invert_(pos_idx >> 0), y = (float)morton3D_invert_(pos_idx >> 1), z = (float)morton3D_invert_(pos_idx >> 2);
		const float rx = rng.next_float(), ry = rng.next_float(), rz = rng.next_float();
		const float sc = scalbnf(1.0f, (int)level);
		V3 p = v3(((x + rx) / (float)GRIDSIZE - 0.5f) * sc + 0.5f, ((y + ry) / (float)GRIDSIZE - 0.5f) * sc + 0.5f, ((z + rz) / (float)GRIDSIZE - 0.5f) * sc + 0.5f);
		V3 pw = warp_position(p, aabb);
		if (u->apply_operators && s->n_ops > 0) {                                               // map_positions, reverse order (:3593-3599)
			bool empty = false;
			map_position_one(s->ops, s->n_ops, pw, empty);
		}
		uint16_t o[16], d16[16];
		network_forward(m, pw, v3(0.5f, 0.5f, 0.5f), o, d16, true);                             // NerfNetwork::density (:3601-3603)
		uint16_t h = f2h(network_to_density(h2f(d16[0]), u->density_activation));               // activate_network_density (:3522-3531)
		uint16_t residual = 0;
		int n_residuals = 0;
		if (u->apply_operators) n_residuals = add_residual_density_one(s->ops, s->n_ops, pw, h, &residual);  // at the MAPPED position (:3612-3620)
		const float ot = h2f(h) * MIN_STEP();                                                   // splat_..._already_activated (:447-463)
		uint32_t ob;
		memcpy(&ob, &ot, 4);
		uint32_t* cell = &tmp[idx];
		uint32_t cur = __atomic_load_n(cell, __ATOMIC_RELAXED);
		while (ob > cur && !__atomic_compare_exchange_n(cell, &cur, ob, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
		if (samples_out) { samples_out[4 * (size_t)i] = pw.x; samples_out[4 * (size_t)i + 1] = pw.y; samples_out[4 * (size_t)i + 2] = pw.z; samples_out[4 * (size_t)i + 3] = h2f(h); }
		if (cells_out) cells_out[i] = idx;
		if (residual_out) residual_out[i] = n_residuals > 1 ? (uint16_t)0x7e00u : residual;
	}
	for (uint32_t i = 0; i < n_cells; ++i) {                                                   // ema_grid_samples_nerf (:483-506)
		float imp;
		memcpy(&imp, &tmp[i], 4);
		float prev = grid[i];
		grid[i] = prev < 0.0f ? prev : fmaxf(prev * u->decay, imp);
	}
	return orc_density_grid_to_bitfield(grid, bits, mean_out);
}

// ---- GrowingSelection::compute_poisson_boundary (growing_selection.cu:2220-2348) on the host --------------------------------
// std::rand() jitter replaced by pcg32(seed) (two draws per sample, u then v), as include/nerfshop_b200.h documents.
// `uniforms` (optional, 2 per sample in (k, i, j) order): the jitter the reference draws with std::rand() (:2245-2246); NULL = seeded pcg32.
int orc_poisson_boundary_ex(const OrcScene* s, const float* points, uint32_t n_points, const NsbBoundarySampling* p, const float* uniforms, float* density_out, float* shs_out,
                         float* coords_out /*optional n*w*w*7*/) {
	Model m;
	if (!model_init(m, &s->desc, s->params, s->n_params)) return 1;
	const uint32_t w = p->sampling_width, n_sh = w * w;
	const Box aabb = mkbox(p->train_aabb_min, p->train_aabb_max);
	Pcg32 rng;
	rng.seed(p->seed, 0xda3e39cb94b95bdbULL);
	std::vector<float> coords((size_t)n_points * n_sh * 7, 0.0f);
	for (uint32_t k = 0; k < n_points; ++k)                                                  // :2238-2260
		for (uint32_t i = 0; i < w; ++i)
			for (uint32_t j = 0; j < w; ++j) {
				const size_t si = (size_t)n_sh * k + (size_t)i * w + j;
				const float ju = uniforms ? uniforms[2 * si] : rng.next_float(), jv = uniforms ? uniforms[2 * si + 1] : rng.next_float();
				float u = ((float)i + ju) / (float)p->hemisphere_width;
				float v = ((float)j + jv) / (float)p->hemisphere_width;
				float theta = (float)(2.f * M_PI * v);
				float phi = acosf(2.f * u - 1.f);
				float x = cosf(theta) * sinf(phi), y = sinf(theta) * sinf(phi), z = cosf(phi);
				float* c = &coords[((size_t)n_sh * k + (size_t)i * w + j) * 7];
				V3 pw = warp_position(v3(points[3 * k], points[3 * k + 1], points[3 * k + 2]), aabb);
				V3 dw = warp_direction(v3(x, y, z));
				c[0] = pw.x; c[1] = pw.y; c[2] = pw.z; c[4] = dw.x; c[5] = dw.y; c[6] = dw.z;
			}
	if (coords_out) memcpy(coords_out, coords.data(), coords.size() * 4);
	const float scale = (float)(4 * M_PI / (double)n_sh);
#pragma omp parallel for schedule(static)
	for (int64_t k = 0; k < (int64_t)n_points; ++k) {
		float sh[27];
		for (int q = 0; q < 27; ++q) sh[q] = 0.0f;
		for (uint32_t i = 0; i < n_sh; ++i) {
			const float* c = &coords[((size_t)n_sh * k + i) * 7];
			uint16_t o[16], d16[16];
			network_forward(m, v3(c[0], c[1], c[2]), v3(c[4], c[5], c[6]), o, d16, false);    // inference_mixed_precision (:2286)
			float rgb[3] = {network_to_rgb(h2f(o[0]), p->rgb_activation), network_to_rgb(h2f(o[1]), p->rgb_activation), network_to_rgb(h2f(o[2]), p->rgb_activation)};
			if (i == 0) {                                                                     // :2325-2327, filter_empty :2200-2218
				float dens = network_to_density(h2f(o[3]), p->density_activation);
				if (p->is_inside) {
					V3 pos = unwarp_position(v3(c[0], c[1], c[2]), aabb);
					int mip = mip_from_pos(pos);
					if (!s->bitfield || !bitfield_at(cascaded_grid_idx_at(pos, (uint32_t)mip), (uint32_t)mip, s->bitfield)) dens = 0.0f;
				}
				density_out[k] = dens;
			}
			V3 d = unwarp_direction(v3(c[4], c[5], c[6]));
			for (int col = 0; col < 3; ++col) {                                               // project_sh9 (sh_utils.cu:30-70), domega = 1
				float* q = sh + 9 * col;
				const float r = rgb[col];
				float cc = 0.282095f;
				q[0] += r * cc * 1.0f;
				cc = 0.488603f;
				q[1] += r * (cc * d.y) * 1.0f;
				q[2] += r * (cc * d.z) * 1.0f;
				q[3] += r * (cc * d.x) * 1.0f;
				cc = 1.092548f;
				q[4] += r * (cc * d.x * d.y) * 1.0f;
				q[5] += r * (cc * d.y * d.z) * 1.0f;
				q[7] += r * (cc * d.x * d.z) * 1.0f;
				cc = 0.315392f;
				q[6] += r * (cc * (3 * d.z * d.z - 1)) * 1.0f;
				cc = 0.546274f;
				q[8] += r * (cc * (d.x * d.x - d.y * d.y)) * 1.0f;
			}
		}
		for (int q = 0; q < 27; ++q) shs_out[(size_t)k * 27 + q] = sh[q] * scale;                // :2341
	}
	return 0;
}
int orc_poisson_boundary(const OrcScene* s, const float* points, uint32_t n_points, const NsbBoundarySampling* p, float* density_out, float* shs_out,
                         float* coords_out /*optional n*w*w*7*/) {
	return orc_poisson_boundary_ex(s, points, n_points, p, nullptr, density_out, shs_out, coords_out);
}
// ---- GrowingSelection::interpolate_poisson_boundary (growing_selection.cu:2350-2398) --------------------------------------
int orc_membrane_blend(const float* gamma, uint32_t n_vertices, uint32_t n_cv, const float* inside_density, const float* outside_density,
                       const float* inside_shs, const float* outside_shs, float* b_shs, float* b_od, float* b_rd) {
	for (uint32_t i = 0; i < n_vertices; ++i) {
		float sum = 0.0f, od = 0.0f, rd = 0.0f, sh[27];
		for (int q = 0; q < 27; ++q) sh[q] = 0.0f;
		for (uint32_t j = 0; j < n_cv; ++j) {
			float alpha_out = 1 - expf(-outside_density[j] * MIN_STEP());
			float alpha_in = 1 - expf(-inside_density[j] * MIN_STEP());
			float w_outside = 1.f;
			float w_inside = std::min(alpha_in / alpha_out, 1.f);
			float g = gamma[(size_t)i * n_cv + j];
			sum += g * alpha_out;
			for (int q = 0; q < 27; ++q) {
				float sh_diff = w_outside * outside_shs[27 * (size_t)j + q] - w_inside * inside_shs[27 * (size_t)j + q];
				sh[q] += g * alpha_out * sh_diff;
			}
			od += g * outside_density[j];
			rd += g * (outside_density[j] - inside_density[j]);
		}
		for (int q = 0; q < 27; ++q) b_shs[27 * (size_t)i + q] = sh[q] / (float)(sum + 1e-6);
		b_od[i] = od;
		b_rd[i] = std::max(rd, 0.f);
	}
	return 0;
}

int orc_set_mlp_policy(int policy) {
	int old = g_mlp_policy;
	if (policy == 0 || policy == 1) g_mlp_policy = policy;
	return old;
}

int orc_set_threads(int n) {
#ifdef _OPENMP
	if (n > 0) omp_set_num_threads(n);
	return omp_get_max_threads();
#else
	(void)n;
	return 1;
#endif
}

} // extern "C"
