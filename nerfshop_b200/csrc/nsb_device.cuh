// nsb_device.cuh — device functions of the render path (sm_90a).
//
// Every fp32 operation that feeds a sample position, a grid index or an fp16 rounding is pinned with
// explicit round-to-nearest intrinsics (__fmul_rn/__fadd_rn/__fmaf_rn/__fdiv_rn) so that ptxas cannot
// re-associate or contract it: the numerics contract of DESIGN.md §3. FMAs appear exactly where nvcc's
// default -fmad=true would contract the reference's own expressions.
// Reference citations are relative to /root/reference (graphdeco-inria/nerfshop).
#pragma once

#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cmath>

#include "../../include/nerfshop_b200.h"

namespace nsb {

// ------------------------------------------------------------------------------------------------
// PODs passed to kernels (kernel-parameter constant bank)
// ------------------------------------------------------------------------------------------------
constexpr int MAX_LEVELS = 16;
constexpr uint32_t GRIDSIZE = 128;
constexpr uint32_t GRIDVOL = 128u * 128u * 128u;
constexpr int CASCADES = 5;
constexpr uint32_t MARCH_ITER = 10000;  // testbed_nerf.cu:56
constexpr int TILE_W = 16, TILE_H = 8;  // ray-init block of the reference (testbed_nerf.cu:2714)
constexpr int TILE_PIXELS = TILE_W * TILE_H;

struct DevLevel {
	float scale;
	uint32_t res;
	uint32_t size;    // entries (2 x fp16 each)
	uint32_t res2;    // res*res (0 for hashed levels)
	uint32_t hashed;  // 1: spatial hash, 0: dense
	uint32_t mask;    // size-1 of a hashed level (a power of two, see build_levels); 0 for dense levels
	const __half2* base;  // first entry of the level (table + level offset): one IMAD.WIDE per gather address
};

struct DevModel {
	DevLevel levels[MAX_LEVELS];
	const __half2* grid;      // hash-grid entries
	const uint8_t* w_image;   // 20480-byte shared-memory image of the 5 weight matrices (wgmma B layout)
	const __half* w_rowmajor; // the same weights, reference order (row-major per layer), for debugging kernels
	uint32_t n_levels;
	uint32_t pair_mode[MAX_LEVELS / 2];  // per pair of levels: 0 both dense, 1 both hashed, 2 mixed
};

struct DevFrame {
	int W, H;
	float fx, fy, cx, cy;
	float cam0[12], cam1[12];
	float rs[4];
	float rmin[3], rmax[3];  // render aabb
	float tmin[3], tmax[3];  // train aabb
	float tinv[3];           // per axis: 1 / (tmax - tmin) when that extent is a power of two (exact), else 0
	int tinv_exact;          // all three tinv are set: warp_position may multiply instead of divide
	float cone, min_T, depth_scale;
	int rgb_act, density_act, mode;
	uint32_t spp;
	float pix_off[2];  // ld_random_pixel_offset(snap ? 0 : spp), pixel independent -> computed on the host
	int apply_ops, poisson_target, linear_colors, min_mip, show_accel;
	int tile_rank, tile_world;
	int tiles_x, tiles_y;
	// ABI 3: the general camera of pixel_to_ray, glow, environment map (all off = the fields above describe the frame completely)
	int general_camera;        // lens distortion, distortion map or depth of field: make_ray_general instead of make_ray
	int cam_dist_mode;         // ECameraDistortionMode
	float cam_dist[7];
	float dof, focus_z;
	int glow_mode;
	float glow_y_cutoff;
	const float* envmap; int env_w, env_h;
	const float* distortion; int dist_w, dist_h;
};

struct DevAffineBox { float mn[3], u[3], v[3], w[3], c[3]; };

struct DevOp {
	int type;
	int copy, apply_poisson, has_poisson_data;
	float amp;
	float amin[3], amax[3];            // scene aabb
	float bmin[3], bmax[3];            // deformed bbox, world
	float wbmin[3], wbmax[3];          // deformed bbox, warped
	float owbmin[3], owbmax[3];        // canonical bbox, warped
	uint32_t n_tets;
	const uint32_t* lut_off;
	const uint32_t* lut_idx;
	const uint32_t* tets;
	const float* verts;
	const float* orig_verts;
	const float* rots;                 // may be null
	const uint8_t* obits;
	const float* shs;                  // 27 per vertex
	const float* od;
	const float* rd;
	DevAffineBox sel, dst;
	float translation[3], scale[3], rot[9];
	int hide_original, correct_dir;
};

// ------------------------------------------------------------------------------------------------
// pinned fp32 arithmetic
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fma_(float a, float b, float c) { return __fmaf_rn(a, b, c); }
__device__ __forceinline__ float div_(float a, float b) { return __fdiv_rn(a, b); }

struct V3 { float x, y, z; };
__device__ __forceinline__ V3 v3(float x, float y, float z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
__device__ __forceinline__ V3 vsub(V3 a, V3 b) { return v3(sub(a.x, b.x), sub(a.y, b.y), sub(a.z, b.z)); }
__device__ __forceinline__ V3 vadd(V3 a, V3 b) { return v3(add(a.x, b.x), add(a.y, b.y), add(a.z, b.z)); }
// Eigen's a.dot(b) reduces as x0*y0 + (x1*y1 + x2*y2) and nvcc contracts that to fma(x0,y0, fma(x1,y1, x2*y2)): the association of
// the reference's own kernels (read off their PTX; the GPU parity tests compare against an nvcc build of those kernels bit for bit)
__device__ __forceinline__ float dot3(V3 a, V3 b) { return fma_(a.x, b.x, fma_(a.y, b.y, mul(a.z, b.z))); }
__device__ __forceinline__ V3 cross3(V3 a, V3 b) {
	return v3(fma_(a.y, b.z, -mul(a.z, b.y)), fma_(a.z, b.x, -mul(a.x, b.z)), fma_(a.x, b.y, -mul(a.y, b.x)));
}
__device__ __forceinline__ V3 madd3(V3 d, float t, V3 o) { return v3(fma_(d.x, t, o.x), fma_(d.y, t, o.y), fma_(d.z, t, o.z)); }
__device__ __forceinline__ V3 ld3(const float* p) { return v3(p[0], p[1], p[2]); }
__device__ __forceinline__ V3 ldv(const float* p, uint32_t i) { return v3(__ldg(p + 3 * i), __ldg(p + 3 * i + 1), __ldg(p + 3 * i + 2)); }

__device__ __forceinline__ float clampf(float v, float lo, float hi) { return v < lo ? lo : (hi < v ? hi : v); }

// ------------------------------------------------------------------------------------------------
// constants — common_nerf.h:16-39
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float MIN_STEP() { return 1.73205080757f / 1024.0f; }
__device__ __forceinline__ float MAX_STEP() { return (1.73205080757f / 1024.0f) * 128.0f; }
__device__ __forceinline__ float DT_RANGE() { return sub(mul(MIN_STEP(), 16.0f), MIN_STEP()); }

// ------------------------------------------------------------------------------------------------
// random_val.cuh:159-322 — Owen-scrambled Sobol, dimension 0 (the only per-pixel use on this path)
// ------------------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t hash_combine(uint32_t seed, uint32_t v) { return seed ^ (v + (seed << 6) + (seed >> 2)); }
__host__ __device__ __forceinline__ uint32_t reverse_bits(uint32_t x) {
#ifdef __CUDA_ARCH__
	return __brev(x);
#else
	x = (((x & 0xaaaaaaaau) >> 1) | ((x & 0x55555555u) << 1));
	x = (((x & 0xccccccccu) >> 2) | ((x & 0x33333333u) << 2));
	x = (((x & 0xf0f0f0f0u) >> 4) | ((x & 0x0f0f0f0fu) << 4));
	x = (((x & 0xff00ff00u) >> 8) | ((x & 0x00ff00ffu) << 8));
	return ((x >> 16) | (x << 16));
#endif
}
__host__ __device__ __forceinline__ uint32_t laine_karras_permutation(uint32_t x, uint32_t seed) {
	x += seed;
	x ^= x * 0x6c50b47cu;
	x ^= x * 0xb82f1e52u;
	x ^= x * 0xc7afe638u;
	x ^= x * 0x8d22f6e6u;
	return x;
}
__host__ __device__ __forceinline__ uint32_t nested_uniform_scramble_base2(uint32_t x, uint32_t seed) {
	return reverse_bits(laine_karras_permutation(reverse_bits(x), seed));
}
// ld_random_val(index, seed, dim = 0): sobol(index, 0) is the bit reversal of index.
__host__ __device__ __forceinline__ float ld_random_val(uint32_t index, uint32_t seed) {
	index = nested_uniform_scramble_base2(index, seed);
	uint32_t x = nested_uniform_scramble_base2(reverse_bits(index), hash_combine(seed, 0));
	return (float)x * 2.3283064365386963e-10f;  // float(1.0/(1ull<<32))
}

// ------------------------------------------------------------------------------------------------
// bounding_box.cuh:180-238
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool box_contains(const float* mn, const float* mx, V3 p) {
	return p.x >= mn[0] && p.x <= mx[0] && p.y >= mn[1] && p.y <= mx[1] && p.z >= mn[2] && p.z <= mx[2];
}
__device__ __forceinline__ float box_ray_tmin(const float* mn, const float* mx, V3 o, V3 d) {
	const float FMAX = 3.402823466e+38f;
	float tmin = div_(sub(mn[0], o.x), d.x), tmax = div_(sub(mx[0], o.x), d.x);
	if (tmin > tmax) { float s = tmin; tmin = tmax; tmax = s; }
	float tymin = div_(sub(mn[1], o.y), d.y), tymax = div_(sub(mx[1], o.y), d.y);
	if (tymin > tymax) { float s = tymin; tymin = tymax; tymax = s; }
	if (tmin > tymax || tymin > tmax) return FMAX;
	if (tymin > tmin) tmin = tymin;
	if (tymax < tmax) tmax = tymax;
	float tzmin = div_(sub(mn[2], o.z), d.z), tzmax = div_(sub(mx[2], o.z), d.z);
	if (tzmin > tzmax) { float s = tzmin; tzmin = tzmax; tzmax = s; }
	if (tmin > tzmax || tzmin > tmax) return FMAX;
	if (tzmin > tmin) tmin = tzmin;
	return tmin;
}

// ------------------------------------------------------------------------------------------------
// common_nerf.cu:5-177
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ V3 warp_position(V3 p, const float* mn, const float* mx) {
	return v3(div_(sub(p.x, mn[0]), sub(mx[0], mn[0])), div_(sub(p.y, mn[1]), sub(mx[1], mn[1])), div_(sub(p.z, mn[2]), sub(mx[2], mn[2])));
}
// warp_position for extents 2^k with the exact inverses 2^-k: (p - mn) / 2^k and (p - mn) * 2^-k are both the correctly rounded value of
// the same real number, subnormals included
__device__ __forceinline__ V3 warp_position_pow2(V3 p, const float* mn, const float* inv) {
	return v3(mul(sub(p.x, mn[0]), inv[0]), mul(sub(p.y, mn[1]), inv[1]), mul(sub(p.z, mn[2]), inv[2]));
}
__device__ __forceinline__ V3 unwarp_position(V3 p, const float* mn, const float* mx) {
	return v3(fma_(p.x, sub(mx[0], mn[0]), mn[0]), fma_(p.y, sub(mx[1], mn[1]), mn[1]), fma_(p.z, sub(mx[2], mn[2]), mn[2]));
}
__device__ __forceinline__ V3 warp_direction(V3 d) { return v3(mul(add(d.x, 1.0f), 0.5f), mul(add(d.y, 1.0f), 0.5f), mul(add(d.z, 1.0f), 0.5f)); }
__device__ __forceinline__ V3 unwarp_direction(V3 d) { return v3(fma_(d.x, 2.0f, -1.0f), fma_(d.y, 2.0f, -1.0f), fma_(d.z, 2.0f, -1.0f)); }
__device__ __forceinline__ float warp_dt(float dt) { return div_(sub(dt, MIN_STEP()), DT_RANGE()); }
__device__ __forceinline__ float unwarp_dt(float dt) { return fma_(dt, DT_RANGE(), MIN_STEP()); }
// t·cone is never NaN (t and cone are finite), and on non-NaN input clamp(x, lo, hi) == min(max(x, lo), hi): two FMNMX
__device__ __forceinline__ float calc_dt(float t, float cone) { return fminf(fmaxf(mul(t, cone), MIN_STEP()), MAX_STEP()); }

// floor(fma(0.5, copysign(1, d), p + 0.5)) is not floor(p) + (d >= 0): p + 0.5 rounds when it crosses a binade (p = 1 - 2^-24 gives 1.5,
// then 2), so the reference's expression is kept as it is
__device__ __forceinline__ float distance_to_next_voxel(V3 pos, V3 dir, V3 idir, uint32_t mip) {  // :93-101
	float fr = __uint_as_float((134u - mip) << 23);  // the cascade's resolution 128 >> mip = 2^(7 - mip), exact
	float px = mul(fr, pos.x), py = mul(fr, pos.y), pz = mul(fr, pos.z);
	float tx = mul(sub(floorf(fma_(0.5f, copysignf(1.0f, dir.x), add(px, 0.5f))), px), idir.x);
	float ty = mul(sub(floorf(fma_(0.5f, copysignf(1.0f, dir.y), add(py, 0.5f))), py), idir.y);
	float tz = mul(sub(floorf(fma_(0.5f, copysignf(1.0f, dir.z), add(pz, 0.5f))), pz), idir.z);
	float t = fminf(fminf(tx, ty), tz);
	return fmaxf(mul(t, __uint_as_float((120u + mip) << 23)), 0.0f);  // fr is a power of two, so t / fr == t * 2^(mip - 7) bit for bit
}
// dt: calc_dt(t, cone), which the caller already has; the reference's do-while computes it again in its first iteration
__device__ __forceinline__ float advance_to_next_voxel(float t, float dt, float cone, V3 pos, V3 dir, V3 idir, uint32_t mip) {  // :103-115
	float t_target = add(t, distance_to_next_voxel(pos, dir, idir, mip));
	t = add(t, dt);
	while (t < t_target) t = add(t, calc_dt(t, cone));
	return t;
}
__host__ __device__ __forceinline__ uint32_t expand_bits(uint32_t v) {
	v = (v * 0x00010001u) & 0xFF0000FFu;
	v = (v * 0x00000101u) & 0x0F00F00Fu;
	v = (v * 0x00000011u) & 0xC30C30C3u;
	v = (v * 0x00000005u) & 0x49249249u;
	return v;
}
__host__ __device__ __forceinline__ uint32_t morton3D(uint32_t x, uint32_t y, uint32_t z) { return expand_bits(x) | (expand_bits(y) << 1) | (expand_bits(z) << 2); }
// expand_bits for v < 128: the first stage, (v * 0x00010001) & 0xFF0000FF, is the identity on such v
__device__ __forceinline__ uint32_t expand_bits7(uint32_t v) {
	v = (v * 0x00000101u) & 0x0F00F00Fu;
	v = (v * 0x00000011u) & 0xC30C30C3u;
	v = (v * 0x00000005u) & 0x49249249u;
	return v;
}
// expand_bits7(i) at index i < 128, for the march kernels' shared-memory copy: three loads replace the three multiply-mask chains
__device__ __forceinline__ void fill_spread7(uint32_t* spread7) {
	for (uint32_t i = threadIdx.x; i < 128; i += blockDim.x) spread7[i] = expand_bits7(i);
}
// the cell coordinates of cascaded_grid_idx_at, each clamped to 0..127
__device__ __forceinline__ void cascaded_grid_coords(V3 pos, uint32_t mip, uint32_t& ix, uint32_t& iy, uint32_t& iz) {  // :117-136
	// fma(a, 2^-mip, 0.5) * 128 == fma(a, 2^(7 - mip), 64) bit for bit: scaling by a power of two commutes with rounding, and
	// neither side can overflow or underflow (|a| is bounded by the AABB; a nonzero sum is a multiple of ulp(a) * 2^-mip >= 2^-29)
	float cell_scale = __uint_as_float((134u - mip) << 23);  // 2^(7 - mip), exact
	float px = fma_(sub(pos.x, 0.5f), cell_scale, 64.0f);
	float py = fma_(sub(pos.y, 0.5f), cell_scale, 64.0f);
	float pz = fma_(sub(pos.z, 0.5f), cell_scale, 64.0f);
	ix = (uint32_t)min(max((int)px, 0), 127); iy = (uint32_t)min(max((int)py, 0), 127); iz = (uint32_t)min(max((int)pz, 0), 127);
}
__device__ __forceinline__ uint32_t cascaded_grid_idx_at(V3 pos, uint32_t mip) {
	uint32_t ix, iy, iz;
	cascaded_grid_coords(pos, mip, ix, iy, iz);
	return expand_bits7(ix) | (expand_bits7(iy) << 1) | (expand_bits7(iz) << 2);
}
// the same index with the 7-bit spread looked up in a fill_spread7 table
__device__ __forceinline__ uint32_t cascaded_grid_idx_at(V3 pos, uint32_t mip, const uint32_t* spread7) {
	uint32_t ix, iy, iz;
	cascaded_grid_coords(pos, mip, ix, iy, iz);
	return spread7[ix] | (spread7[iy] << 1) | (spread7[iz] << 2);
}
__device__ __forceinline__ bool bitfield_at(uint32_t idx, uint32_t mip, const uint8_t* __restrict__ bf) {
	return (__ldg(bf + (idx >> 3) + mip * (GRIDVOL / 8)) & (1u << (idx & 7u))) != 0;
}
__device__ __forceinline__ int mip_from_pos(V3 pos) {  // :163-168
	float maxval = fmaxf(fmaxf(fabsf(sub(pos.x, 0.5f)), fabsf(sub(pos.y, 0.5f))), fabsf(sub(pos.z, 0.5f)));
	// clamp(frexp exponent + 1, 0, 4) from the exponent field e of maxval >= 0: a normal maxval gives e - 126 + 1; a subnormal has e = 0 and
	// a frexp exponent <= -126, both clamp to 0; maxval == 0 (the exact AABB centre) is frexpf(0) + 1 = 1
	const uint32_t b = __float_as_uint(maxval);
	return b == 0 ? 1 : min(CASCADES - 1, max(0, (int)(b >> 23) - 125));
}
__device__ __forceinline__ int mip_from_dt(float dt, V3 pos) {  // :170-177
	int mip = mip_from_pos(pos);
	dt = mul(dt, 256.0f);
	// dt >= 1 is normal, so its frexp exponent is (bits >> 23) - 126; below 1 the position's mip stands
	const int e = dt < 1.0f ? 0 : (int)(__float_as_uint(dt) >> 23) - 126;
	return min(CASCADES - 1, max(e, mip));
}
__device__ __forceinline__ float logistic_(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float network_to_rgb(float v, int act) {  // :38-47
	switch (act) {
		case 0: return v;
		case 1: return v > 0.0f ? v : 0.0f;
		case 2: return logistic_(v);
		default: return __expf(clampf(v, -10.0f, 10.0f));
	}
}
__device__ __forceinline__ float network_to_density(float v, int act) {  // :57-66
	switch (act) {
		case 0: return v;
		case 1: return v > 0.0f ? v : 0.0f;
		case 2: return logistic_(v);
		default: return __expf(v);
	}
}
__device__ __forceinline__ float srgb_to_linear(float s) {  // common_device.cuh:31-37
	if (s <= 0.04045f) return s / 12.92f;
	return powf((s + 0.055f) / 1.055f, 2.4f);
}

// ------------------------------------------------------------------------------------------------
// ray generation — init_rays_with_payload_kernel_nerf (testbed_nerf.cu:2512-2616) + pixel_to_ray
// (common_device.cuh:245-295, dof = 0, no distortion) and the march loop shared by advance_pos_nerf
// (:588-603) and generate_next_nerf_network_inputs (:671-688)
// ------------------------------------------------------------------------------------------------
struct Ray { V3 o, d; float t; };

__device__ __forceinline__ V3 matvec3(const float* M, V3 v) {  // column-major 3x3 (first 9 floats)
	return v3(fma_(M[0], v.x, fma_(M[3], v.y, mul(M[6], v.z))), fma_(M[1], v.x, fma_(M[4], v.y, mul(M[7], v.z))),
	          fma_(M[2], v.x, fma_(M[5], v.y, mul(M[8], v.z))));
}
__device__ __forceinline__ V3 matTvec3(const float* M, V3 v) {
	return v3(fma_(M[0], v.x, fma_(M[1], v.y, mul(M[2], v.z))), fma_(M[3], v.x, fma_(M[4], v.y, mul(M[5], v.z))),
	          fma_(M[6], v.x, fma_(M[7], v.y, mul(M[8], v.z))));
}

// returns false when the ray misses the render AABB (payload.alive = false at :2591-2595)
__device__ __forceinline__ bool make_ray(const DevFrame& f, uint32_t px, uint32_t py, Ray& r) {
	uint32_t idx = px + (uint32_t)f.W * py;
	float fw = (float)f.W, fh = (float)f.H;
	float u = mul(add((float)px, 0.5f), div_(1.0f, fw));
	float v = mul(add((float)py, 0.5f), div_(1.0f, fh));
	float rt = fma_(f.rs[1], u, f.rs[0]);
	rt = fma_(f.rs[2], v, rt);
	if (f.rs[3] != 0.0f) rt = fma_(f.rs[3], ld_random_val(f.spp, idx * 72239731u), rt);
	else rt = fma_(0.0f, 0.0f, rt);
	float cam[12];
	float omrt = sub(1.0f, rt);
#pragma unroll
	for (int i = 0; i < 12; ++i) cam[i] = fma_(f.cam0[i], rt, mul(f.cam1[i], omrt));
	float uvx = div_(add((float)px, f.pix_off[0]), fw);
	float uvy = div_(add((float)py, f.pix_off[1]), fh);
	V3 dl = v3(div_(mul(sub(uvx, f.cx), fw), f.fx), div_(mul(sub(uvy, f.cy), fh), f.fy), 1.0f);
	V3 d = matvec3(cam, dl);
	r.o = v3(cam[9], cam[10], cam[11]);
	float n2 = dot3(d, d);
	if (n2 > 0.0f) { float n = __fsqrt_rn(n2); d = v3(div_(d.x, n), div_(d.y, n), div_(d.z, n)); }
	r.d = d;
	float t = add(fmaxf(box_ray_tmin(f.rmin, f.rmax, r.o, r.d), 0.05f), 1e-6f);
	if (!box_contains(f.rmin, f.rmax, madd3(r.d, t, r.o))) return false;
	r.t = t;
	return true;
}

// ------------------------------------------------------------------------------------------------
// The general camera: pixel_to_ray with lens distortion, a distortion map and depth of field (common_device.cuh:79-110,145-295),
// square2disk_shirley / ld_random_val_2d (random_val.cuh:109-127,278-282). Only k_prepare_rays<true> / k_march_trace<true> contain it: frames that
// ask for it hand the persistent renderer their rays through a side buffer; plain fp32 with the compiler's own contraction, like the reference's: these frames are held to the
// 1e-3 frame tolerance, not to bit-exact ray generation (Newton iterations, sincosf).
// ------------------------------------------------------------------------------------------------
__device__ const uint32_t c_sobol_dir1[32] = {
	0x80000000u, 0xc0000000u, 0xa0000000u, 0xf0000000u, 0x88000000u, 0xcc000000u, 0xaa000000u, 0xff000000u, 0x80800000u, 0xc0c00000u, 0xa0a00000u,
	0xf0f00000u, 0x88880000u, 0xcccc0000u, 0xaaaa0000u, 0xffff0000u, 0x80008000u, 0xc000c000u, 0xa000a000u, 0xf000f000u, 0x88008800u, 0xcc00cc00u,
	0xaa00aa00u, 0xff00ff00u, 0x80808080u, 0xc0c0c0c0u, 0xa0a0a0a0u, 0xf0f0f0f0u, 0x88888888u, 0xccccccccu, 0xaaaaaaaau, 0xffffffffu,
};
__device__ __forceinline__ void ld_random_val_2d(uint32_t index, uint32_t seed, float& x, float& y) {
	index = nested_uniform_scramble_base2(index, seed);
	uint32_t X1 = 0;
	for (uint32_t bit = 0; bit < 32; ++bit) X1 ^= ((index >> bit) & 1u) * c_sobol_dir1[bit];
	x = (float)nested_uniform_scramble_base2(reverse_bits(index), hash_combine(seed, 0)) * 2.3283064365386963e-10f;
	y = (float)nested_uniform_scramble_base2(X1, hash_combine(seed, 1)) * 2.3283064365386963e-10f;
}
__device__ __forceinline__ void apply_camera_distortion(const float* p, float u, float v, float& du, float& dv) {  // :145-160
	const float k1 = p[0], k2 = p[1], p1 = p[2], p2 = p[3];
	const float u2 = u * u, uv = u * v, v2 = v * v, r2 = u2 + v2;
	const float radial = k1 * r2 + k2 * r2 * r2;
	du = u * radial + 2.0f * p1 * uv + p2 * (r2 + 2.0f * u2);
	dv = v * radial + 2.0f * p2 * uv + p1 * (r2 + 2.0f * v2);
}
__device__ __forceinline__ void iterative_camera_undistortion(const float* params, float& u, float& v) {  // :163-197
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
// read_image<2> (:79-110): bilinear, clamped, position in [0,1]^2 scaled by (resolution - 1)
__device__ __forceinline__ void read_image2(const float* __restrict__ data, int rw, int rh, float px, float py, float& ox, float& oy) {
	const float fx = px * (float)(rw - 1), fy = py * (float)(rh - 1);
	const int tx = (int)fx, ty = (int)fy;
	const float wx = fx - (float)tx, wy = fy - (float)ty;
	auto rd = [&](int x, int y) { x = max(min(x, rw - 1), 0); y = max(min(y, rh - 1), 0); return *reinterpret_cast<const float2*>(data + 2 * ((size_t)x + (size_t)y * rw)); };
	const float2 a = rd(tx, ty), b = rd(tx + 1, ty), c = rd(tx, ty + 1), d = rd(tx + 1, ty + 1);
	ox = (1.0f - wx) * (1.0f - wy) * a.x + wx * (1.0f - wy) * b.x + (1.0f - wx) * wy * c.x + wx * wy * d.x;
	oy = (1.0f - wx) * (1.0f - wy) * a.y + wx * (1.0f - wy) * b.y + (1.0f - wx) * wy * c.y + wx * wy * d.y;
}
// read_envmap (envmap.cuh:30-62): latitude-longitude map, bilinear, wraps in x, clamps in y
__device__ __forceinline__ float4 read_envmap(const float* __restrict__ data, int rw, int rh, V3 dir) {
	// dir_to_spherical_unorm({dir.z, -dir.x, dir.y}) (random_val.cuh:64-69)
	const float cos_theta = fminf(fmaxf(dir.y, -1.0f), 1.0f);
	const float theta = acosf(cos_theta);
	const float phi = atan2f(-dir.x, dir.z);
	const float cyl_x = theta / 3.14159265358979323846f, cyl_y = phi / (2.0f * 3.14159265358979323846f) + 0.5f;
	const float ex = cyl_y * (float)(rw - 1), ey = cyl_x * (float)(rh - 1);
	const int tx = (int)ex, ty = (int)ey;
	const float wx = ex - (float)tx, wy = ey - (float)ty;
	auto rd = [&](int x, int y) {
		if (x < 0) x += rw; else if (x >= rw) x -= rw;
		y = max(min(y, rh - 1), 0);
		return *reinterpret_cast<const float4*>(data + 4 * ((size_t)x + (size_t)y * rw));
	};
	const float4 a = rd(tx, ty), b = rd(tx + 1, ty), c = rd(tx, ty + 1), d = rd(tx + 1, ty + 1);
	const float w00 = (1.0f - wx) * (1.0f - wy), w10 = wx * (1.0f - wy), w01 = (1.0f - wx) * wy, w11 = wx * wy;
	return make_float4(w00 * a.x + w10 * b.x + w01 * c.x + w11 * d.x, w00 * a.y + w10 * b.y + w01 * c.y + w11 * d.y,
	                   w00 * a.z + w10 * b.z + w01 * c.z + w11 * d.z, w00 * a.w + w10 * b.w + w01 * c.w + w11 * d.w);
}
// init_rays_with_payload_kernel_nerf (:2546-2595) with the general pixel_to_ray. r.o / r.d are valid even when the ray misses the AABB (the
// environment map is looked up for every pixel).
__device__ __forceinline__ bool make_ray_general(const DevFrame& f, uint32_t px, uint32_t py, Ray& r) {
	const uint32_t idx = px + (uint32_t)f.W * py;
	const float fw = (float)f.W, fh = (float)f.H;
	const float u = ((float)px + 0.5f) * (1.0f / fw), v = ((float)py + 0.5f) * (1.0f / fh);
	const float rt = f.rs[0] + f.rs[1] * u + f.rs[2] * v + f.rs[3] * ld_random_val(f.spp, idx * 72239731u);
	float cam[12];
#pragma unroll
	for (int i = 0; i < 12; ++i) cam[i] = f.cam0[i] * rt + f.cam1[i] * (1.0f - rt);
	const float uvx = ((float)px + f.pix_off[0]) / fw, uvy = ((float)py + f.pix_off[1]) / fh;
	V3 dl;
	if (f.cam_dist_mode == 2) {  // f_theta_undistortion (:232-245)
		const float xpix = (uvx - f.cx) * f.cam_dist[5], ypix = (uvy - f.cy) * f.cam_dist[6];
		const float norm = sqrtf(xpix * xpix + ypix * ypix);
		const float alpha = f.cam_dist[0] + norm * (f.cam_dist[1] + norm * (f.cam_dist[2] + norm * (f.cam_dist[3] + norm * f.cam_dist[4])));
		float sa, ca;
		sincosf(alpha, &sa, &ca);
		if (ca <= 1.17549435e-38f || norm == 0.0f) {  // the reference returns a ray outside the AABB: the pixel is not rendered
			r.o = v3(1000.0f, 0.0f, 0.0f);
			r.d = v3(0.0f, 0.0f, 1.0f);
			return false;
		}
		sa *= 1.0f / norm;
		dl = v3(sa * xpix, sa * ypix, ca);
	} else {
		dl = v3((uvx - f.cx) * fw / f.fx, (uvy - f.cy) * fh / f.fy, 1.0f);
		if (f.cam_dist_mode == 1) iterative_camera_undistortion(f.cam_dist, dl.x, dl.y);
	}
	if (f.distortion) {
		float ox, oy;
		read_image2(f.distortion, f.dist_w, f.dist_h, uvx, uvy, ox, oy);
		dl.x += ox; dl.y += oy;
	}
	V3 d = matvec3(cam, dl);
	V3 o = v3(cam[9], cam[10], cam[11]);
	if (f.dof != 0.0f) {
		const V3 lookat = v3(o.x + d.x * f.focus_z, o.y + d.y * f.focus_z, o.z + d.z * f.focus_z);
		float sx, sy;
		ld_random_val_2d(f.spp, px * 19349663u + py * 96925573u, sx, sy);
		const float a = sx * 2.0f - 1.0f, b = sy * 2.0f - 1.0f;  // square2disk_shirley
		float rr, phi;
		if (a * a > b * b) { rr = a; phi = (3.14159265358979323846f / 4.0f) * (b / a); }
		else { rr = b; phi = (3.14159265358979323846f / 2.0f) - (3.14159265358979323846f / 4.0f) * (a / b); }
		float sp, cp;
		sincosf(phi, &sp, &cp);
		const float bx = f.dof * (rr * cp), by = f.dof * (rr * sp);
		o = v3(o.x + (cam[0] * bx + cam[3] * by), o.y + (cam[1] * bx + cam[4] * by), o.z + (cam[2] * bx + cam[5] * by));
		d = v3((lookat.x - o.x) / f.focus_z, (lookat.y - o.y) / f.focus_z, (lookat.z - o.z) / f.focus_z);
	}
	const float n2 = d.x * d.x + d.y * d.y + d.z * d.z;
	if (n2 > 0.0f) { const float n = sqrtf(n2); d = v3(d.x / n, d.y / n, d.z / n); }
	r.o = o;
	r.d = d;
	const float t = add(fmaxf(box_ray_tmin(f.rmin, f.rmax, o, d), 0.05f), 1e-6f);
	if (!box_contains(f.rmin, f.rmax, madd3(d, t, o))) return false;
	r.t = t;
	return true;
}

// glow_mode of composite_kernel_nerf (:807-903): grid-line visualisation added to (or replacing) a sample's colour; `weight_mask` multiplies the
// sample's weight (mask_to_alpha). pos = the sample's unwarped position, cam_origin = camera_matrix.col(3). Everything by value (an array
// passed by address would move the caller's colour into local memory on the hot path): returns {r, g, b, weight mask}.
__device__ __noinline__ float4 glow_apply(int glow_mode, float glow_y_cutoff, V3 pos, V3 cam_origin, float r_in, float g_in, float b_in) {
	float rgb[3] = {r_in, g_in, b_in};
	float weight_mask = 1.0f;
	float glow = 0.0f;
	const bool green_grid = glow_mode & 1, green_cutline = glow_mode & 2, mask_to_alpha = glow_mode & 4, radial_mode = glow_mode & 8, grid_mode = glow_mode & 16;
	float dist;
	if (radial_mode) {
		const V3 q = vsub(pos, cam_origin);
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
#pragma unroll 1
		for (int k = 0; k < 4; ++k) {
			const float m = (float)(2 << k);  // 2, 4, 8, 16
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
	return make_float4(rgb[0], rgb[1], rgb[2], weight_mask);
}

// Next occupied sample at or after t. false: the ray left the render AABB.
// spread7: the block's fill_spread7 table in shared memory
__device__ __forceinline__ bool next_occupied(const DevFrame& f, const uint8_t* __restrict__ bitfield, const uint32_t* spread7, V3 o, V3 d, V3 idir,
                                              float& t, float& dt, V3& pos, uint32_t& mip_out, uint32_t& cell_out) {
	while (true) {
		pos = madd3(d, t, o);
		if (!box_contains(f.rmin, f.rmax, pos)) return false;
		dt = calc_dt(t, f.cone);
		uint32_t mip = (uint32_t)max(f.min_mip, mip_from_dt(dt, pos));
		uint32_t cell = cascaded_grid_idx_at(pos, mip, spread7);
		if (!bitfield || bitfield_at(cell, mip, bitfield)) { mip_out = mip; cell_out = cell; return true; }
		t = advance_to_next_voxel(t, dt, f.cone, pos, d, idir, mip);
	}
}

// The same walk, resumable: at most `budget` empty voxels are skipped per call. The state of the walk is `t`
// alone (always a point of the ray's dt lattice), so splitting it over several calls yields bit-identical samples.
enum MarchResult { MARCH_FOUND = 0, MARCH_EXIT = 1, MARCH_PENDING = 2 };
__device__ __forceinline__ MarchResult next_occupied_budget(const DevFrame& f, const uint8_t* __restrict__ bitfield, const uint32_t* spread7, V3 o, V3 d, V3 idir,
                                                            float& t, float& dt, V3& pos, int& budget) {
	while (true) {
		pos = madd3(d, t, o);
		if (!box_contains(f.rmin, f.rmax, pos)) return MARCH_EXIT;
		dt = calc_dt(t, f.cone);
		uint32_t mip = (uint32_t)max(f.min_mip, mip_from_dt(dt, pos));
		uint32_t cell = cascaded_grid_idx_at(pos, mip, spread7);
		if (!bitfield || bitfield_at(cell, mip, bitfield)) return MARCH_FOUND;
		if (budget <= 0) return MARCH_PENDING;
		--budget;
		t = advance_to_next_voxel(t, dt, f.cone, pos, d, idir, mip);
	}
}

// ------------------------------------------------------------------------------------------------
// tiny-cuda-nn GridEncoding (HashGrid, F = 2, linear) — SURVEY.md Appendix B.
// One level: 8 gathers of a __half2, result += (half)(weight * data) with fp16 accumulation.
// ------------------------------------------------------------------------------------------------
// tcnn grid_index: dense levels index x + y*res + z*res^2, the others hash the vertex (primes 1, 2654435761, 805459861); then `% size`,
// on the uint32 index, for every grid coordinate (positions outside [0,1]^3 wrap the coordinates through uint32).
// MODE 0: dense, 1: hashed, 2: either (level kind is uniform across the launch: a select, not a divergent branch).
// IN_RANGE: the caller guarantees every coordinate is at most res (a warped position in [-0.5/scale, 1 + 0.5/scale] and a model whose
// dense levels satisfy dense_in_range), so a dense index is below res + res^2 + res^3 < 2*size and one conditional subtraction is the
// modulo. Only the fused renderer's frames without operators whose render AABB lies inside the train AABB take it (render_in_range).
__host__ __device__ __noinline__ inline uint32_t grid_mod_slow(uint32_t d, uint32_t size) { return d % size; }
template <int MODE, bool IN_RANGE = false>
__host__ __device__ __forceinline__ uint32_t grid_index(const DevLevel& L, uint32_t gx, uint32_t gy, uint32_t gz) {
	uint32_t h = 0, d = 0;
	if (MODE != 0) {
		h = gx ^ (gy * 2654435761u) ^ (gz * 805459861u);
		h &= L.mask;  // tcnn's `index % size`: a hashed level's size is a power of two (build_levels)
	}
	if (MODE != 1) {
		d = gx + gy * L.res + gz * L.res2;
		// `index % size` (dense size <= 2^24, so 2*size does not wrap). The division sits behind a branch in a call that is not inlined,
		// so it is never if-converted into the gather loop: in-cube samples pay a compare and a branch.
		if (IN_RANGE) d = d >= L.size ? d - L.size : d;
		else d = d < L.size ? d : (d < 2u * L.size ? d - L.size : grid_mod_slow(d, L.size));
	}
	return MODE == 0 ? d : (MODE == 1 ? h : (L.hashed ? h : d));
}

// NL consecutive levels at once: all 8*NL gathers are issued before the first one is consumed (memory-level parallelism;
// the walk is bound by L1/L2 gather throughput, not by arithmetic).
template <int NL, int MODE, bool IN_RANGE = false>
__device__ __forceinline__ void encode_levels(const DevLevel* __restrict__ L, const __half2* __restrict__ grid, float x, float y, float z, __half2* out) {
	__half2 v[NL][8];
	float wx[NL], wy[NL], wz[NL];
#pragma unroll
	for (int l = 0; l < NL; ++l) {
		float px = fma_(L[l].scale, x, 0.5f), py = fma_(L[l].scale, y, 0.5f), pz = fma_(L[l].scale, z, 0.5f);
		float fx = floorf(px), fy = floorf(py), fz = floorf(pz);
		wx[l] = sub(px, fx); wy[l] = sub(py, fy); wz[l] = sub(pz, fz);
		// (int) is cvt.rzi.s32.f32, as in tcnn: truncation, NaN -> 0, saturation outside the int range (the oracle's cvt_rzi_s32)
		uint32_t gx = (uint32_t)(int)fx, gy = (uint32_t)(int)fy, gz = (uint32_t)(int)fz;
		const __half2* base = L[l].base;
#pragma unroll
		for (int c = 0; c < 8; ++c) v[l][c] = __ldg(base + grid_index<MODE, IN_RANGE>(L[l], gx + (c & 1), gy + ((c >> 1) & 1), gz + ((c >> 2) & 1)));
	}
#pragma unroll
	for (int l = 0; l < NL; ++l) {
		float ax[2] = {sub(1.0f, wx[l]), wx[l]}, ay[2] = {sub(1.0f, wy[l]), wy[l]}, az[2] = {sub(1.0f, wz[l]), wz[l]};
		__half2 acc = __floats2half2_rn(0.0f, 0.0f);
#pragma unroll
		for (int c = 0; c < 8; ++c) {
			float w = mul(mul(ax[c & 1], ay[(c >> 1) & 1]), az[(c >> 2) & 1]);
			float2 d = __half22float2(v[l][c]);
			acc = __hadd2(acc, __floats2half2_rn(mul(w, d.x), mul(w, d.y)));  // result += (T)(weight * data), fp16 accumulate
		}
		out[l] = acc;
	}
}
__device__ __forceinline__ __half2 encode_level(const DevLevel& L, const __half2* __restrict__ grid, float x, float y, float z) {
	__half2 out;
	encode_levels<1, 2>(&L, grid, x, y, z, &out);
	return out;
}

// tcnn SphericalHarmonics degree 4 on 2*d-1 -> 16 fp16 packed as 8 half2
__device__ __forceinline__ void encode_sh4(V3 dw, __half2* out) {
	float x = fma_(dw.x, 2.0f, -1.0f), y = fma_(dw.y, 2.0f, -1.0f), z = fma_(dw.z, 2.0f, -1.0f);
	float xy = mul(x, y), xz = mul(x, z), yz = mul(y, z), x2 = mul(x, x), y2 = mul(y, y), z2 = mul(z, z);
	float o[16];
	o[0] = 0.28209479177387814f;
	o[1] = mul(-0.48860251190291987f, y);
	o[2] = mul(0.48860251190291987f, z);
	o[3] = mul(-0.48860251190291987f, x);
	o[4] = mul(1.0925484305920792f, xy);
	o[5] = mul(-1.0925484305920792f, yz);
	o[6] = sub(mul(0.94617469575755997f, z2), 0.31539156525251999f);
	o[7] = mul(-1.0925484305920792f, xz);
	o[8] = sub(mul(0.54627421529603959f, x2), mul(0.54627421529603959f, y2));
	o[9] = mul(mul(0.59004358992664352f, y), add(mul(-3.0f, x2), y2));
	o[10] = mul(mul(2.8906114426405538f, xy), z);
	o[11] = mul(mul(0.45704579946446572f, y), sub(1.0f, mul(5.0f, z2)));
	o[12] = mul(mul(0.3731763325901154f, z), sub(mul(5.0f, z2), 3.0f));
	o[13] = mul(mul(0.45704579946446572f, x), sub(1.0f, mul(5.0f, z2)));
	o[14] = mul(mul(1.4453057213202769f, z), sub(x2, y2));
	o[15] = mul(mul(0.59004358992664352f, x), add(-x2, mul(3.0f, y2)));
#pragma unroll
	for (int i = 0; i < 8; ++i) out[i] = __floats2half2_rn(o[2 * i], o[2 * i + 1]);
}

// ------------------------------------------------------------------------------------------------
// tcnn::default_rng_t = pcg32 (M. O'Neill's PCG-XSH-RR 64/32, public algorithm; tiny-cuda-nn pcg32.h [tcnn-ext]);
// used by generate_grid_samples_nerf_nonuniform (common_nerf.cu:179-208).
// ------------------------------------------------------------------------------------------------
struct Pcg32 {
	uint64_t state, inc;
	__host__ __device__ __forceinline__ uint32_t next_uint() {
		uint64_t old = state;
		state = old * 0x5851f42d4c957f2dULL + inc;
		uint32_t xorshifted = (uint32_t)(((old >> 18u) ^ old) >> 27u);
		uint32_t rot = (uint32_t)(old >> 59u);
		return (xorshifted >> rot) | (xorshifted << ((~rot + 1u) & 31u));
	}
	__device__ __forceinline__ float next_float() { return sub(__uint_as_float((next_uint() >> 9) | 0x3f800000u), 1.0f); }
	__host__ __device__ __forceinline__ void advance(uint64_t delta) {  // LCG skip-ahead in O(log delta)
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

// ------------------------------------------------------------------------------------------------
// editing — selection_utils.h:10-47, cage_deformation.cu:197-269,431-541, affine_duplication.cu:92-118
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float scalar_tp(V3 a, V3 b, V3 c) { return dot3(a, cross3(b, c)); }
__device__ __forceinline__ bool same_side_tet(V3 v1, V3 v2, V3 v3_, V3 v4, V3 p) {
	V3 normal = cross3(vsub(v2, v1), vsub(v3_, v1));
	float dotV4 = dot3(normal, vsub(v4, v1));
	float dotP = dot3(normal, vsub(p, v1));
	return (__float_as_uint(dotV4) >> 31) == (__float_as_uint(dotP) >> 31);
}
__device__ __forceinline__ bool point_in_tet(V3 a, V3 b, V3 c, V3 d, V3 p) {
	return same_side_tet(a, b, c, d, p) && same_side_tet(b, c, d, a, p) && same_side_tet(c, d, a, b, p) && same_side_tet(d, a, b, c, p);
}
__device__ __forceinline__ void bary_tet(V3 a, V3 b, V3 c, V3 d, V3 p, float* out) {
	V3 vap = vsub(p, a), vbp = vsub(p, b), vab = vsub(b, a), vac = vsub(c, a), vad = vsub(d, a), vbc = vsub(c, b), vbd = vsub(d, b);
	float va6 = scalar_tp(vbp, vbd, vbc);
	float vb6 = scalar_tp(vap, vac, vad);
	float vc6 = scalar_tp(vap, vad, vab);
	float vd6 = scalar_tp(vap, vab, vac);
	float v6 = (float)__drcp_rn((double)scalar_tp(vab, vac, vad));  // "1. / x": double division, then float
	out[0] = mul(va6, v6); out[1] = mul(vb6, v6); out[2] = mul(vc6, v6); out[3] = mul(vd6, v6);
}
__device__ __forceinline__ float bary_mix1(const float* b, float a0, float a1, float a2, float a3) {
	return fma_(b[3], a3, fma_(b[2], a2, fma_(b[0], a0, mul(b[1], a1))));  // ((b0*a0 + b1*a1) + b2*a2) + b3*a3 as nvcc contracts it
}
__device__ __forceinline__ V3 bary_mix(const float* b, V3 a0, V3 a1, V3 a2, V3 a3) {
	return v3(bary_mix1(b, a0.x, a1.x, a2.x, a3.x), bary_mix1(b, a0.y, a1.y, a2.y, a3.y), bary_mix1(b, a0.z, a1.z, a2.z, a3.z));
}
// first tet of the sample's cell list that contains p (cage_deformation.cu:221-248); -1 if none
__device__ __forceinline__ int find_tet(const DevOp& op, V3 p, float* bary) {
	int level = mip_from_pos(p);
	uint32_t cell = (uint32_t)level * GRIDVOL + cascaded_grid_idx_at(p, (uint32_t)level);
	uint32_t j0 = __ldg(op.lut_off + cell), j1 = __ldg(op.lut_off + cell + 1);
	for (uint32_t j = j0; j < j1; ++j) {
		uint32_t t = __ldg(op.lut_idx + j);
		uint4 tv = __ldg(reinterpret_cast<const uint4*>(op.tets) + t);
		V3 a = ldv(op.verts, tv.x), b = ldv(op.verts, tv.y), c = ldv(op.verts, tv.z), d = ldv(op.verts, tv.w);
		if (point_in_tet(a, b, c, d, p)) { bary_tet(a, b, c, d, p, bary); return (int)t; }
	}
	return -1;
}
__device__ __forceinline__ void cage_map(const DevOp& op, V3& pw, V3& dw, bool& empty) {  // interpolate_tet
	if (op.n_tets == 0) return;
	bool in_deformed = false;
	if (box_contains(op.wbmin, op.wbmax, pw)) {
		V3 p = unwarp_position(pw, op.amin, op.amax);
		float b[4];
		int t = find_tet(op, p, b);
		if (t >= 0) {
			uint4 tv = __ldg(reinterpret_cast<const uint4*>(op.tets) + t);
			V3 canon = bary_mix(b, ldv(op.orig_verts, tv.x), ldv(op.orig_verts, tv.y), ldv(op.orig_verts, tv.z), ldv(op.orig_verts, tv.w));
			pw = warp_position(canon, op.amin, op.amax);
			if (op.rots) {
				float R[9];
#pragma unroll
				for (int k = 0; k < 9; ++k) R[k] = __ldg(op.rots + 9 * (size_t)t + k);
				dw = warp_direction(matvec3(R, unwarp_direction(dw)));
			}
			in_deformed = true;
		}
	}
	if (!op.copy && !in_deformed && box_contains(op.owbmin, op.owbmax, pw)) {
		V3 p = unwarp_position(pw, op.amin, op.amax);
		int level = mip_from_pos(p);
		if (bitfield_at(cascaded_grid_idx_at(p, (uint32_t)level), (uint32_t)level, op.obits)) empty = true;
	}
}
__device__ __forceinline__ bool abox_contains(const DevAffineBox& b, V3 p) {
	V3 q = vsub(p, ld3(b.mn));
	V3 u = ld3(b.u), v = ld3(b.v), w = ld3(b.w);
	float du = dot3(u, q), dv = dot3(v, q), dw = dot3(w, q);
	return du >= 0 && du < dot3(u, u) && dv >= 0 && dv < dot3(v, v) && dw >= 0 && dw < dot3(w, w);
}
__device__ __forceinline__ void affine_map(const DevOp& op, V3& pw, V3& dw, bool& empty) {  // translate_in_box
	if (abox_contains(op.dst, pw)) {
		V3 c = ld3(op.dst.c);
		V3 q = vsub(pw, c);
		q = v3(div_(q.x, op.scale[0]), div_(q.y, op.scale[1]), div_(q.z, op.scale[2]));
		V3 r = matTvec3(op.rot, q);
		pw = vsub(vadd(r, c), ld3(op.translation));
		if (op.correct_dir) dw = warp_direction(matTvec3(op.rot, unwarp_direction(dw)));
	} else if (op.hide_original && abox_contains(op.sel, pw)) {
		empty = true;
	}
}
__device__ __forceinline__ void map_one(const DevOp* __restrict__ ops, int n_ops, V3& pw, V3& dw, bool& empty) {
	for (int i = n_ops - 1; i >= 0; --i) {  // reverse list order (testbed_nerf.cu:2899)
		if (ops[i].type == 0) cage_map(ops[i], pw, dw, empty);
		else affine_map(ops[i], pw, dw, empty);
	}
}
// compute_residual_poisson_kernel for one sample: which op/tet/barycentrics supply the membrane data.
struct Membrane { int op; int tet; float b[4]; float dob, drb; };
__device__ __forceinline__ void poisson_one(const DevOp* __restrict__ ops, int n_ops, V3 pw, Membrane& m) {
	m.op = -1; m.tet = -1; m.dob = 0.0f; m.drb = 0.0f;
	for (int i = n_ops - 1; i >= 0; --i) {  // testbed_nerf.cu:2868; a later (lower-index) operator overwrites
		const DevOp& op = ops[i];
		if (op.type != 0 || !op.apply_poisson || !op.has_poisson_data || op.n_tets == 0) continue;
		V3 p = unwarp_position(pw, op.amin, op.amax);
		if (!box_contains(op.bmin, op.bmax, p)) continue;
		float b[4];
		int t = find_tet(op, p, b);
		if (t < 0) continue;
		uint4 tv = __ldg(reinterpret_cast<const uint4*>(op.tets) + t);
		float od = bary_mix1(b, __ldg(op.od + tv.x), __ldg(op.od + tv.y), __ldg(op.od + tv.z), __ldg(op.od + tv.w));
		float rd = bary_mix1(b, __ldg(op.rd + tv.x), __ldg(op.rd + tv.y), __ldg(op.rd + tv.z), __ldg(op.rd + tv.w));
		m.op = i; m.tet = t;
		m.b[0] = b[0]; m.b[1] = b[1]; m.b[2] = b[2]; m.b[3] = b[3];
		m.dob = mul(op.amp, od);
		m.drb = mul(op.amp, rd);
	}
}
// boundary_shs interpolated at the sample (cage_deformation.cu:485-488), coefficient k of 27
__device__ __forceinline__ float membrane_sh(const DevOp* __restrict__ ops, const Membrane& m, int k) {
	const DevOp& op = ops[m.op];
	uint4 tv = __ldg(reinterpret_cast<const uint4*>(op.tets) + m.tet);
	return bary_mix1(m.b, __ldg(op.shs + 27 * (size_t)tv.x + k), __ldg(op.shs + 27 * (size_t)tv.y + k),
	                 __ldg(op.shs + 27 * (size_t)tv.z + k), __ldg(op.shs + 27 * (size_t)tv.w + k));
}
// evaluate_sh9 (common_nerf.cu:218-245) of the interpolated membrane SH
__device__ __forceinline__ void membrane_rgb(const DevOp* __restrict__ ops, const Membrane& m, V3 d, float* rgb) {
	float p[9];
	float z2 = mul(d.z, d.z);
	p[0] = 0.2820947917738781f;
	p[2] = mul(0.4886025119029199f, d.z);
	p[6] = fma_(0.9461746957575601f, z2, -0.3153915652525201f);
	p[3] = mul(-0.48860251190292f, d.x);
	p[1] = mul(-0.48860251190292f, d.y);
	float tb = mul(-1.092548430592079f, d.z);
	p[7] = mul(tb, d.x);
	p[5] = mul(tb, d.y);
	float c1 = fma_(d.x, d.x, -mul(d.y, d.y));
	float s1 = fma_(d.x, d.y, mul(d.y, d.x));
	p[8] = mul(0.5462742152960395f, c1);
	p[4] = mul(0.5462742152960395f, s1);
	for (int c = 0; c < 3; ++c) {
		float acc = mul(p[0], membrane_sh(ops, m, c * 9 + 0));
		for (int k = 1; k < 9; ++k) acc = fma_(p[k], membrane_sh(ops, m, c * 9 + k), acc);
		rgb[c] = acc;
	}
}

// ------------------------------------------------------------------------------------------------
// Level table of the hash grid (host). Shared with the host build of grid_index that the CPU tests compile.
// ------------------------------------------------------------------------------------------------
// Accepted: the configs/nerf/base.json topology, log2_hashmap_size 1..24, base_resolution >= 1, per_level_scale >= 1 (not NaN) and every
// level's scale below 2^32, so that tcnn's `(uint32_t)ceilf(scale) + 1` resolution is defined and fits a uint32.
inline bool build_levels(const NsbModelDesc* d, DevLevel* L, uint64_t* n_grid_entries) {
	if (!d || d->n_levels != 16 || d->n_features_per_level != 2 || d->n_neurons != 64 || d->n_hidden_density != 1 || d->n_hidden_rgb != 2 ||
	    d->sh_degree != 4 || d->log2_hashmap_size == 0 || d->log2_hashmap_size > 24 || d->base_resolution == 0 || !(d->per_level_scale >= 1.0f))
		return false;
	float l2s = log2f(d->per_level_scale);
	uint64_t offset = 0;
	for (uint32_t l = 0; l < d->n_levels; ++l) {
		float scale = exp2f((float)l * l2s) * (float)d->base_resolution - 1.0f;  // tcnn grid_scale
		if (!(scale < 4294967296.0f)) return false;                                // also rejects inf
		uint32_t res = (uint32_t)ceilf(scale) + 1u;                                // tcnn grid_resolution
		double dense = (double)res * res * res;
		uint32_t max_params = 0xffffffffu / 2;
		uint32_t n = dense > (double)max_params ? max_params : (uint32_t)dense;
		n = ((n + 7u) / 8u) * 8u;
		n = n < (1u << d->log2_hashmap_size) ? n : (1u << d->log2_hashmap_size);
		// tcnn's grid_index decides hash vs. dense with a uint32 stride: `for (dim < 3 && stride <= size) stride *= res`, hashed iff
		// size < stride. The stride can wrap (res = 2^18 at aabb_scale 128: res^2 = 2^36 = 0 mod 2^32), and then tcnn indexes the level densely.
		uint32_t stride = 1;
		for (int dim = 0; dim < 3 && stride <= n; ++dim) stride *= res;
		L[l].scale = scale;
		L[l].res = res;
		L[l].base = reinterpret_cast<const __half2*>((uintptr_t)offset * sizeof(__half2));  // entry offset; rebased onto the table by nsb_upload_model
		L[l].size = n;
		L[l].hashed = n < stride ? 1u : 0u;
		L[l].res2 = L[l].hashed ? 0u : res * res;  // tcnn's third stride, uint32
		// Hashed implies size = 2^log2_hashmap_size: size < stride <= res^3 with no wrap means the cap was taken; a wrap means res^3 > 2^32
		// and the cap as well. So mask = size - 1, and grid_index takes a hashed level's `index % size` as `index & mask`.
		L[l].mask = L[l].hashed ? n - 1 : 0u;
		offset += n;
	}
	*n_grid_entries = offset;
	return true;
}

// grid_index<MODE, true>'s condition for in-cube positions (coordinates at most res): every dense level's index stays below 2*size.
inline bool dense_in_range(const DevLevel* L, uint32_t n_levels) {
	for (uint32_t l = 0; l < n_levels; ++l) {
		if (L[l].hashed) continue;
		const uint64_t r = L[l].res;
		if (r * r * r >= (1ull << 32) || r + r * r + r * r * r >= 2ull * L[l].size) return false;
	}
	return true;
}

}  // namespace nsb
