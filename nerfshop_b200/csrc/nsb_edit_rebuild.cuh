// nsb_edit_rebuild.cuh — the per-EDIT level of the cage scheme on the device (SURVEY.md §8f-1).
// Included by nsb_kernels.cu (same translation unit: it needs NsbContext and DevOp).
//
// The reference rebuilds a dragged cage on the host with 32 threads and re-uploads a 42 MB offsets array per drag:
//   Cage::interpolate_with_mvc        (src/editing/datastructures/cage.cu:39-55)      tet vertices = MVC weights x cage vertices
//   TetMesh::post_update_vertices     (src/editing/datastructures/tet_mesh.cu:13-20)  bounding boxes
//   TetMesh::update_local_rotations   (tet_mesh.cu:38-74)                             per-tet Kabsch rotation
//   TetMesh::build_tet_grid           (tet_mesh.cu:369-667)                           per-cell tet lists (CSR) over 5 x 128^3 cells
// Here the operator's arrays never leave HBM: one call takes the new cage vertices (a few hundred bytes) and rebuilds the
// vertex array, rotations, boxes and the CSR in place. The cell predicates repeat nsb_host_geometry.cpp's arithmetic
// (plain, non-contracted fp32: every product and sum rounded separately, as gcc emits it for x86-64 without FMA), so the
// device CSR is bit-identical to the host one; tests/test_gpu_edit_rebuild.py asserts exactly that.
#pragma once
#include "nsb_kabsch.h"

namespace nsb {
namespace rebuild {

struct P3 { float x, y, z; };
__device__ __forceinline__ P3 p3(float x, float y, float z) { P3 r; r.x = x; r.y = y; r.z = z; return r; }
__device__ __forceinline__ P3 psub(P3 a, P3 b) { return p3(sub(a.x, b.x), sub(a.y, b.y), sub(a.z, b.z)); }
__device__ __forceinline__ float pdot(P3 a, P3 b) { return add(add(mul(a.x, b.x), mul(a.y, b.y)), mul(a.z, b.z)); }
__device__ __forceinline__ P3 pcross(P3 a, P3 b) {
	return p3(sub(mul(a.y, b.z), mul(a.z, b.y)), sub(mul(a.z, b.x), mul(a.x, b.z)), sub(mul(a.x, b.y), mul(a.y, b.x)));
}
__device__ __forceinline__ P3 pld(const float* v, uint32_t i) { return p3(v[3 * i], v[3 * i + 1], v[3 * i + 2]); }
__device__ __forceinline__ bool sign_of(float v) { return (__float_as_uint(v) >> 31) != 0; }
__device__ __forceinline__ bool same_side(P3 v1, P3 v2, P3 v3, P3 v4, P3 p) {  // selection_utils.h:33-47
	P3 n = pcross(psub(v2, v1), psub(v3, v1));
	return sign_of(pdot(n, psub(v4, v1))) == sign_of(pdot(n, psub(p, v1)));
}
__device__ __forceinline__ bool point_in_tet(const P3* v, P3 p) {
	return same_side(v[0], v[1], v[2], v[3], p) && same_side(v[1], v[2], v[3], v[0], p) && same_side(v[2], v[3], v[0], v[1], p) &&
	       same_side(v[3], v[0], v[1], v[2], p);
}
__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (hi < v ? hi : v); }
__device__ __forceinline__ float pow2f(int e) { return __uint_as_float((uint32_t)(127 + e) << 23); }
// selection_utils.cu:65-83
__device__ __forceinline__ P3 get_cell_pos(uint32_t x, uint32_t y, uint32_t z, uint32_t level) {
	const float s = pow2f((int)level);
	return p3(add(mul(sub(div_(add((float)x, 0.5f), 128.0f), 0.5f), s), 0.5f), add(mul(sub(div_(add((float)y, 0.5f), 128.0f), 0.5f), s), 0.5f),
	          add(mul(sub(div_(add((float)z, 0.5f), 128.0f), 0.5f), s), 0.5f));
}
__device__ __forceinline__ void get_cell_at_pos(P3 pos, uint32_t level, int* out) {
	const float s = pow2f(-(int)level);
	out[0] = clampi((int)mul(add(mul(sub(pos.x, 0.5f), s), 0.5f), 128.0f), 0, 127);
	out[1] = clampi((int)mul(add(mul(sub(pos.y, 0.5f), s), 0.5f), 128.0f), 0, 127);
	out[2] = clampi((int)mul(add(mul(sub(pos.z, 0.5f), s), 0.5f), 128.0f), 0, 127);
}
__device__ __forceinline__ void project(const P3* pts, int n, P3 axis, float& mn, float& mx) {
	mn = INFINITY; mx = -INFINITY;
	for (int i = 0; i < n; ++i) {
		float v = pdot(axis, pts[i]);
		if (v < mn) mn = v;
		if (v > mx) mx = v;
	}
}
// BoundingBox::intersects(Triangle): separating-axis test (bounding_box.cuh:126-178)
__device__ __forceinline__ bool box_intersects_triangle(P3 bmin, P3 bmax, P3 a, P3 b, P3 c) {
	float tmin, tmax, bmn, bmx;
	const P3 bn[3] = {p3(1, 0, 0), p3(0, 1, 0), p3(0, 0, 1)};
	const float bminv[3] = {bmin.x, bmin.y, bmin.z}, bmaxv[3] = {bmax.x, bmax.y, bmax.z};
	P3 tri[3] = {a, b, c};
	for (int i = 0; i < 3; ++i) {
		project(tri, 3, bn[i], tmin, tmax);
		if (tmax < bminv[i] || tmin > bmaxv[i]) return false;
	}
	P3 verts[8] = {p3(bmin.x, bmin.y, bmin.z), p3(bmin.x, bmin.y, bmax.z), p3(bmin.x, bmax.y, bmin.z), p3(bmin.x, bmax.y, bmax.z),
	               p3(bmax.x, bmin.y, bmin.z), p3(bmax.x, bmin.y, bmax.z), p3(bmax.x, bmax.y, bmin.z), p3(bmax.x, bmax.y, bmax.z)};
	P3 n = pcross(psub(b, a), psub(c, a));
	float len = __fsqrt_rn(pdot(n, n));
	if (len > 0.0f) n = p3(div_(n.x, len), div_(n.y, len), div_(n.z, len));
	float off = pdot(n, a);
	project(verts, 8, n, bmn, bmx);
	if (bmx < off || bmn > off) return false;
	const P3 edges[3] = {psub(a, b), psub(a, c), psub(b, c)};
	for (int i = 0; i < 3; ++i)
		for (int j = 0; j < 3; ++j) {
			P3 axis = pcross(edges[i], bn[j]);
			project(verts, 8, axis, bmn, bmx);
			project(tri, 3, axis, tmin, tmax);
			if (bmx < tmin || bmn > tmax) return false;
		}
	return true;
}

// ---- Cage::interpolate_with_mvc: one thread per tet-mesh vertex, the host's sequential fp32 accumulation order -------------------
__global__ void k_mvc_apply(const float* __restrict__ W, uint32_t n_points, uint32_t n_cv, const float* __restrict__ cage, float* __restrict__ out) {
	extern __shared__ float s_cage[];  // 3 * n_cv
	for (uint32_t k = threadIdx.x; k < 3 * n_cv; k += blockDim.x) s_cage[k] = cage[k];
	__syncthreads();
	uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
	if (p >= n_points) return;
	float ax = 0.0f, ay = 0.0f, az = 0.0f;
	const float* w = W + (size_t)p * n_cv;
	for (uint32_t v = 0; v < n_cv; ++v) {
		float wv = __ldg(w + v);
		ax = add(ax, mul(wv, s_cage[3 * v]));
		ay = add(ay, mul(wv, s_cage[3 * v + 1]));
		az = add(az, mul(wv, s_cage[3 * v + 2]));
	}
	out[3 * p] = ax; out[3 * p + 1] = ay; out[3 * p + 2] = az;
}

// ---- TetMesh::post_update_vertices: boxes of the deformed vertices; out = {bbox min, bbox max, warped min, warped max} -----------
__global__ void k_cage_bbox(const float* __restrict__ verts, uint32_t n, const float* __restrict__ aabb /*min3,max3*/, float* __restrict__ out) {
	__shared__ float smn[3][256], smx[3][256];
	float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
	for (uint32_t i = threadIdx.x; i < n; i += blockDim.x)
		for (int k = 0; k < 3; ++k) { float v = verts[3 * i + k]; mn[k] = fminf(mn[k], v); mx[k] = fmaxf(mx[k], v); }
	for (int k = 0; k < 3; ++k) { smn[k][threadIdx.x] = mn[k]; smx[k][threadIdx.x] = mx[k]; }
	__syncthreads();
	for (int s = 128; s > 0; s >>= 1) {
		if ((int)threadIdx.x < s)
			for (int k = 0; k < 3; ++k) {
				smn[k][threadIdx.x] = fminf(smn[k][threadIdx.x], smn[k][threadIdx.x + s]);
				smx[k][threadIdx.x] = fmaxf(smx[k][threadIdx.x], smx[k][threadIdx.x + s]);
			}
		__syncthreads();
	}
	if (threadIdx.x < 3) {
		const int k = threadIdx.x;
		out[k] = smn[k][0];
		out[3 + k] = smx[k][0];
		const float ext = sub(aabb[3 + k], aabb[k]);
		out[6 + k] = div_(sub(smn[k][0], aabb[k]), ext);
		out[9 + k] = div_(sub(smx[k][0], aabb[k]), ext);
	}
}

// ---- TetMesh::update_local_rotations: proper Kabsch rotation per tet, in double (nsb_kabsch.h) ---------------------------------------
__global__ void k_local_rotations(const float* __restrict__ verts, const float* __restrict__ orig, const uint32_t* __restrict__ tets, uint32_t n_tets,
                                  float* __restrict__ rots) {
	uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= n_tets) return;
	tet_rotation(verts, orig, tets + 4 * (size_t)t, rots + 9 * (size_t)t);
}

// ---- the cell box of one (tet, cascade) and the cell test of build_tet_grid and vanish (tet_mesh.cu:278-330, :407-460) -------------
// Loads tet t's vertices into v and returns the number of cells of its box at `level`: first cell lo, extents (.., ny, nz), half cell
// size h. (v stays a separate array: the face loop indexes it dynamically, so it lives in local memory, and nothing else should.)
__device__ __forceinline__ uint32_t tet_cell_box(const float* __restrict__ verts, const uint32_t* __restrict__ tets, uint32_t t, uint32_t level, P3* v, int* lo,
                                                 uint32_t& ny, uint32_t& nz, float& h) {
	for (int j = 0; j < 4; ++j) v[j] = pld(verts, tets[4 * t + j]);
	P3 mn = v[0], mx = v[0];
	for (int j = 1; j < 4; ++j) {
		mn = p3(fminf(mn.x, v[j].x), fminf(mn.y, v[j].y), fminf(mn.z, v[j].z));
		mx = p3(fmaxf(mx.x, v[j].x), fmaxf(mx.y, v[j].y), fmaxf(mx.z, v[j].z));
	}
	int hi[3];
	get_cell_at_pos(mn, level, lo);
	get_cell_at_pos(mx, level, hi);
	const uint32_t nx = (uint32_t)(hi[0] - lo[0] + 1);
	ny = (uint32_t)(hi[1] - lo[1] + 1);
	nz = (uint32_t)(hi[2] - lo[2] + 1);
	const uint32_t n_cells = nx * ny * nz;
	const float scale = pow2f((int)level);
	h = div_(mul(0.5f, scale), 128.0f);
	return n_cells;
}
// Cell c of the box: its coordinates, and whether the tet touches it (a cell corner inside the tet, or a tet face hitting the cell box).
__device__ __forceinline__ bool tet_touches_cell(const P3* v, const int* lo, uint32_t ny, uint32_t nz, float h, uint32_t c, uint32_t level, uint32_t& x,
                                                 uint32_t& y, uint32_t& z) {
	x = (uint32_t)lo[0] + c / (ny * nz); y = (uint32_t)lo[1] + (c / nz) % ny; z = (uint32_t)lo[2] + c % nz;
	const P3 ctr = get_cell_pos(x, y, z, level);
	bool inside = false;
#pragma unroll 1
	for (int k = 0; k < 8 && !inside; ++k) {
		// corner order of the host code; +-0.5 * scale / 128 is exact
		const float sx = (k == 3 || k == 4 || k == 6 || k == 7) ? h : -h;
		const float sy = (k == 2 || k == 4 || k == 5 || k == 7) ? h : -h;
		const float sz = (k == 1 || k == 5 || k == 6 || k == 7) ? h : -h;
		inside = point_in_tet(v, p3(add(ctr.x, sx), add(ctr.y, sy), add(ctr.z, sz)));
	}
	if (!inside) {
		const P3 bmin = p3(sub(ctr.x, h), sub(ctr.y, h), sub(ctr.z, h)), bmax = p3(add(ctr.x, h), add(ctr.y, h), add(ctr.z, h));
#pragma unroll 1
		for (int j = 0; j < 4 && !inside; ++j) inside = box_intersects_triangle(bmin, bmax, v[j], v[(j + 1) & 3], v[(j + 2) & 3]);
	}
	return inside;
}

// ---- TetMesh::build_tet_grid, pass 1: one CTA per (tet, cascade); its threads stride over the cells of the tet's box -----------
struct Mark { uint32_t cell, tet; };
__global__ void __launch_bounds__(128) k_tet_mark(const float* __restrict__ verts, const uint32_t* __restrict__ tets, uint32_t n_tets, uint32_t* __restrict__ counts,
                                                  Mark* __restrict__ marks, uint32_t marks_cap, unsigned int* __restrict__ n_marks) {
	const uint32_t t = blockIdx.x / CASCADES, level = blockIdx.x % CASCADES;
	if (t >= n_tets) return;
	P3 v[4];
	int lo[3];
	uint32_t ny, nz;
	float h;
	const uint32_t n_cells = tet_cell_box(verts, tets, t, level, v, lo, ny, nz, h);
	for (uint32_t c = threadIdx.x; c < n_cells; c += blockDim.x) {
		uint32_t x, y, z;
		if (tet_touches_cell(v, lo, ny, nz, h, c, level, x, y, z)) {
			const uint32_t cell = level * GRIDVOL + morton3D(x, y, z);
			atomicAdd(counts + cell, 1u);
			const unsigned int pos = atomicAdd(n_marks, 1u);
			if (pos < marks_cap) { marks[pos].cell = cell; marks[pos].tet = t; }
		}
	}
}

// ---- TetMesh::vanish (tet_mesh.cu:251-363) and clear_grid (:239-248): k_tet_mark's launch shape and cell test ------------------
// Every touched cell's density becomes 0 (grid may be null) and its occupancy bit is cleared with an atomicAnd on the 32-bit word that
// holds it: many CTAs clear bits of one word, where the reference clears from one thread. Clearing is idempotent, so a cell touched by
// several tets needs no dedup. A counted call (n_cleared != null) with a grid takes two launches so that each changed cell counts once:
// the first (mark_nonzero) zeroes the densities and SETS the bit of every cell whose density was not 0, the second (grid == null) clears
// the bits and counts those it found set.
__global__ void __launch_bounds__(128) k_tet_vanish(const float* __restrict__ verts, const uint32_t* __restrict__ tets, uint32_t n_tets, float* __restrict__ grid,
                                                    uint32_t* __restrict__ bits, int mark_nonzero, unsigned long long* __restrict__ n_cleared) {
	const uint32_t t = blockIdx.x / CASCADES, level = blockIdx.x % CASCADES;
	if (t >= n_tets) return;
	P3 v[4];
	int lo[3];
	uint32_t ny, nz;
	float h;
	const uint32_t n_cells = tet_cell_box(verts, tets, t, level, v, lo, ny, nz, h);
	uint32_t n = 0;
	for (uint32_t c = threadIdx.x; c < n_cells; c += blockDim.x) {
		uint32_t x, y, z;
		if (!tet_touches_cell(v, lo, ny, nz, h, c, level, x, y, z)) continue;
		const uint32_t cell = level * GRIDVOL + morton3D(x, y, z), mask = 1u << (cell & 31u);  // byte cell/8, bit cell%8 = word cell/32, bit cell%32
		if (mark_nonzero) {
			if (__float_as_uint(atomicExch(grid + cell, 0.0f)) != 0u) atomicOr(bits + (cell >> 5), mask);
			continue;
		}
		if (grid) grid[cell] = 0.0f;
		if (n_cleared) n += (atomicAnd(bits + (cell >> 5), ~mask) & mask) != 0u;
		else atomicAnd(bits + (cell >> 5), ~mask);
	}
	if (n) atomicAdd(n_cleared, (unsigned long long)n);
}

// ---- exclusive scan of the per-cell counts (3 launches: block sums, scan of block sums, block scans + offset) -------------------
constexpr uint32_t SCAN_ITEMS = 4, SCAN_THREADS = 1024, SCAN_TILE = SCAN_ITEMS * SCAN_THREADS;
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* total) {  // 1024 threads
	__shared__ uint32_t warp_sums[32];
	const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
	uint32_t inc = v;
	for (int o = 1; o < 32; o <<= 1) { uint32_t n = __shfl_up_sync(0xffffffffu, inc, o); if ((int)lane >= o) inc += n; }
	if (lane == 31) warp_sums[warp] = inc;
	__syncthreads();
	if (warp == 0) {
		uint32_t w = warp_sums[lane], winc = w;
		for (int o = 1; o < 32; o <<= 1) { uint32_t n = __shfl_up_sync(0xffffffffu, winc, o); if ((int)lane >= o) winc += n; }
		warp_sums[lane] = winc - w;  // exclusive
		if (lane == 31 && total) *total = winc;
	}
	__syncthreads();
	uint32_t r = inc - v + warp_sums[warp];
	__syncthreads();
	return r;
}
__global__ void __launch_bounds__(1024) k_scan_block_sums(const uint32_t* __restrict__ counts, uint32_t n, uint32_t* __restrict__ block_sums) {
	const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
	uint32_t s = 0;
	for (uint32_t k = 0; k < SCAN_ITEMS; ++k) if (base + k < n) s += counts[base + k];
	__shared__ uint32_t total;
	block_exclusive_scan(s, &total);
	if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}
__global__ void __launch_bounds__(1024) k_scan_sums(uint32_t* __restrict__ block_sums, uint32_t n_blocks, uint32_t* __restrict__ grand_total) {
	// n_blocks <= 1024 * 4
	const uint32_t base = threadIdx.x * SCAN_ITEMS;
	uint32_t v[SCAN_ITEMS], s = 0;
	for (uint32_t k = 0; k < SCAN_ITEMS; ++k) { v[k] = base + k < n_blocks ? block_sums[base + k] : 0u; s += v[k]; }
	__shared__ uint32_t total;
	uint32_t ex = block_exclusive_scan(s, &total);
	for (uint32_t k = 0; k < SCAN_ITEMS; ++k) { if (base + k < n_blocks) block_sums[base + k] = ex; ex += v[k]; }
	if (threadIdx.x == 0) *grand_total = total;
}
__global__ void __launch_bounds__(1024) k_scan_apply(const uint32_t* __restrict__ counts, uint32_t n, const uint32_t* __restrict__ block_sums,
                                                     const uint32_t* __restrict__ grand_total, uint32_t* __restrict__ offsets) {
	const uint32_t base = blockIdx.x * SCAN_TILE + threadIdx.x * SCAN_ITEMS;
	uint32_t v[SCAN_ITEMS], s = 0;
	for (uint32_t k = 0; k < SCAN_ITEMS; ++k) { v[k] = base + k < n ? counts[base + k] : 0u; s += v[k]; }
	uint32_t ex = block_exclusive_scan(s, nullptr) + block_sums[blockIdx.x];
	for (uint32_t k = 0; k < SCAN_ITEMS; ++k) { if (base + k < n) offsets[base + k] = ex; ex += v[k]; }
	if (blockIdx.x == 0 && threadIdx.x == 0) offsets[n] = *grand_total;
}
// ---- pass 2: scatter the marks into their cells, then order each cell's list by tet index (the host's generation order) ---------
__global__ void k_tet_fill(const Mark* __restrict__ marks, uint32_t n_marks, const uint32_t* __restrict__ offsets, uint32_t* __restrict__ counts,
                           uint32_t* __restrict__ idx) {
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_marks) return;
	const Mark m = marks[i];
	const uint32_t k = atomicSub(counts + m.cell, 1u) - 1u;
	idx[offsets[m.cell] + k] = m.tet;
}
// Lists of up to SORT_SHORT tets (fine cascades) are ordered by their own thread; longer ones (coarse cascades: one cell can hold
// every tet of the mesh) are queued for k_tet_sort_long.
constexpr uint32_t SORT_SHORT = 24, SORT_SMEM = 8192;
__global__ void k_tet_sort(const uint32_t* __restrict__ offsets, uint32_t n_cells, uint32_t* __restrict__ idx, uint32_t* __restrict__ long_cells,
                           unsigned int* __restrict__ n_long) {
	uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
	if (c >= n_cells) return;
	const uint32_t j0 = offsets[c], j1 = offsets[c + 1];
	if (j1 - j0 > SORT_SHORT) { long_cells[atomicAdd(n_long, 1u)] = c; return; }
	for (uint32_t a = j0 + 1; a < j1; ++a) {  // insertion sort
		const uint32_t key = idx[a];
		uint32_t b = a;
		while (b > j0 && idx[b - 1] > key) { idx[b] = idx[b - 1]; --b; }
		idx[b] = key;
	}
}
// One CTA per long list: bitonic sort on a power-of-two buffer padded with 0xffffffff — in shared memory up to SORT_SMEM
// entries, else in `scratch` at [2*j0, 2*j0 + P) (P < 2L, so the regions of different cells are disjoint; scratch holds 2 * n_idx words).
__global__ void __launch_bounds__(256) k_tet_sort_long(const uint32_t* __restrict__ offsets, uint32_t* __restrict__ idx, const uint32_t* __restrict__ long_cells,
                                                       const unsigned int* __restrict__ n_long, uint32_t* __restrict__ scratch) {
	__shared__ uint32_t sm[SORT_SMEM];
	const uint32_t n = *n_long;
	for (uint32_t b = blockIdx.x; b < n; b += gridDim.x) {
		const uint32_t c = long_cells[b];
		const uint32_t j0 = offsets[c], L = offsets[c + 1] - j0;
		uint32_t P = 1;
		while (P < L) P <<= 1;
		uint32_t* buf = P <= SORT_SMEM ? sm : scratch + 2 * (size_t)j0;
		for (uint32_t i = threadIdx.x; i < P; i += blockDim.x) buf[i] = i < L ? idx[j0 + i] : 0xffffffffu;
		__syncthreads();
		for (uint32_t k = 2; k <= P; k <<= 1)
			for (uint32_t j = k >> 1; j > 0; j >>= 1) {
				for (uint32_t t = threadIdx.x; t < (P >> 1); t += blockDim.x) {
					const uint32_t i = ((t & ~(j - 1)) << 1) | (t & (j - 1));  // lower index of the pair, partner = i + j
					const uint32_t x = buf[i], y = buf[i + j];
					const bool up = (i & k) == 0;
					if ((x > y) == up) { buf[i] = y; buf[i + j] = x; }
				}
				__syncthreads();
			}
		for (uint32_t i = threadIdx.x; i < L; i += blockDim.x) idx[j0 + i] = buf[i];
		__syncthreads();
	}
}

// ---- GrowingSelection::compute_poisson_boundary, device part: activate_network_output (:2182-2198), filter_empty (:2200-2218)
// and the SH9 Monte-Carlo fit (:2334-2344, project_sh9 sh_utils.cu:30-70). One CTA per point; thread (col, k) owns coefficient k of
// colour col and accumulates the samples in order, like the host loop. net: fp16 [16 x n_padded] row-major from the inference kernel.
__global__ void __launch_bounds__(32) k_boundary_fit(const __half* __restrict__ net, uint32_t n_padded, const float* __restrict__ coords, uint32_t n_sh,
                                                     int rgb_act, int density_act, const uint8_t* __restrict__ bitfield, const float* __restrict__ aabb,
                                                     float scale, float* __restrict__ density_out, float* __restrict__ shs_out) {
	const uint32_t pt = blockIdx.x, tid = threadIdx.x;
	const uint32_t s0 = pt * n_sh;
	if (tid == 31) {
		float dens = network_to_density(__half2float(net[(size_t)3 * n_padded + s0]), density_act);
		if (bitfield) {  // is_inside
			V3 p = unwarp_position(v3(coords[7 * (size_t)s0], coords[7 * (size_t)s0 + 1], coords[7 * (size_t)s0 + 2]), aabb, aabb + 3);
			int mip = mip_from_pos(p);
			if (!bitfield_at(cascaded_grid_idx_at(p, (uint32_t)mip), (uint32_t)mip, bitfield)) dens = 0.0f;
		}
		density_out[pt] = dens;
	}
	if (tid >= 27) return;
	const uint32_t col = tid / 9, k = tid % 9;
	float acc = 0.0f;
	for (uint32_t i = 0; i < n_sh; ++i) {
		const size_t s = (size_t)s0 + i;
		const float rgb = network_to_rgb(__half2float(net[(size_t)col * n_padded + s]), rgb_act);
		const V3 d = unwarp_direction(v3(coords[7 * s + 4], coords[7 * s + 5], coords[7 * s + 6]));
		float basis;
		switch (k) {  // float constants, products left to right as the reference writes them
			case 0: basis = 0.282095f; break;
			case 1: basis = mul(0.488603f, d.y); break;
			case 2: basis = mul(0.488603f, d.z); break;
			case 3: basis = mul(0.488603f, d.x); break;
			case 4: basis = mul(mul(1.092548f, d.x), d.y); break;
			case 5: basis = mul(mul(1.092548f, d.y), d.z); break;
			case 7: basis = mul(mul(1.092548f, d.x), d.z); break;
			case 6: basis = mul(0.315392f, sub(mul(mul(3.0f, d.z), d.z), 1.0f)); break;
			default: basis = mul(0.546274f, sub(mul(d.x, d.x), mul(d.y, d.y))); break;
		}
		acc = add(acc, mul(mul(rgb, basis), 1.0f));
	}
	shs_out[(size_t)pt * 27 + tid] = mul(acc, scale);
}

// ---- GrowingSelection::interpolate_poisson_boundary (:2350-2398): thread (tet vertex, coefficient slot); slots 0-26 the SH entries,
// 27 the outside density, 28 the residual density. alpha_out/alpha_in/w_inside per cage vertex come from the host (libm expf).
__global__ void k_membrane_blend(const float* __restrict__ gamma, uint32_t n_vertices, uint32_t n_cv, const float* __restrict__ alpha_out,
                                 const float* __restrict__ w_inside, const float* __restrict__ d_in, const float* __restrict__ d_out,
                                 const float* __restrict__ shs_in, const float* __restrict__ shs_out_, float* __restrict__ b_shs, float* __restrict__ b_od,
                                 float* __restrict__ b_rd) {
	const uint32_t i = blockIdx.x * blockDim.y + threadIdx.y, slot = threadIdx.x;
	if (i >= n_vertices || slot >= 29) return;
	const float* g = gamma + (size_t)i * n_cv;
	if (slot < 27) {
		float acc = 0.0f, wsum = 0.0f;
		for (uint32_t j = 0; j < n_cv; ++j) {
			const float sh_diff = sub(mul(1.0f, shs_out_[27 * (size_t)j + slot]), mul(w_inside[j], shs_in[27 * (size_t)j + slot]));
			const float ga = mul(g[j], alpha_out[j]);
			wsum = add(wsum, ga);
			acc = add(acc, mul(ga, sh_diff));
		}
		b_shs[27 * (size_t)i + slot] = div_(acc, (float)((double)wsum + 1e-6));
	} else if (slot == 27) {
		float acc = 0.0f;
		for (uint32_t j = 0; j < n_cv; ++j) acc = add(acc, mul(g[j], d_out[j]));
		b_od[i] = acc;
	} else {
		float acc = 0.0f;
		for (uint32_t j = 0; j < n_cv; ++j) acc = add(acc, mul(g[j], sub(d_out[j], d_in[j])));
		b_rd[i] = fmaxf(acc, 0.0f);
	}
}

}  // namespace rebuild
}  // namespace nsb
