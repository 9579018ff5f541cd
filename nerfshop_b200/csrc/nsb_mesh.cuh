// Mesh extraction on the device: the kernels behind nsb_density_on_grid, nsb_marching_cubes and nsb_mesh_shade.
// Included by nsb_kernels.cu after the network kernels (network_tiles, linear_to_srgb).
//
//   k_density_on_grid      Testbed::get_density_on_grid (testbed_nerf.cu:4538-4586): generate_grid_samples_nerf_uniform (:402-413)
//                          + NerfNetwork::density + grid_samples_half_to_float (:465-481) in one pass, no position buffer
//   k_mc_count / k_mc_scan / k_mc_vertices / k_mc_faces
//                          marching_cubes_gpu (marching_cubes.cu:730-758) with gen_vertices' arithmetic (:217-265), made deterministic:
//                          vertices ordered by (grid point, axis x/y/z), triangles by (cell, table row order)
//   k_mesh_degree / k_mesh_fill / k_mesh_normals
//                          the normal half of accumulate_1ring (:267-302) summed per vertex in triangle order, without float atomics
//   k_mesh_colors          generate_nerf_network_inputs_from_positions (testbed_nerf.cu:608-614) + NerfNetwork::inference
//                          + extract_srgb_with_activation (:338-351)
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>
#include <cub/device/device_scan.cuh>

#include "nsb_mc_table.h"

namespace mesh {

__device__ const int8_t kMcTri[256][NSB_MC_ROW] = NSB_MC_TRI_TABLE_INIT;
__device__ const uint8_t kMcCount[256] = NSB_MC_TRI_COUNT_INIT;

constexpr uint32_t THREADS = 256;
constexpr uint32_t PER_THREAD = 4;
constexpr uint32_t TILE = THREADS * PER_THREAD;  // grid points per CTA of the marching-cubes passes

struct GridQuery {
	uint32_t res[3];
	float inv_res[3];  // 1.f / res, as generate_grid_samples_nerf_uniform computes it
	float rmin[3], rext[3];  // the AABB meshed: min and max - min
	float tmin[3], tmax[3];  // the train AABB (m_aabb)
};

// ---- density on a grid ---------------------------------------------------------------------------------------------
// Grid point i of the query, x fastest: pos = x * (1/res) * (max - min) + min, with the product and sum contracted into one FMA as
// nvcc compiles the reference's Eigen expression.
__device__ __forceinline__ V3 grid_point(const GridQuery& q, uint32_t i) {
	const uint32_t rxy = q.res[0] * q.res[1];
	const uint32_t z = i / rxy, r = i - z * rxy, y = r / q.res[0], x = r - y * q.res[0];
	return v3(fma_(mul((float)x, q.inv_res[0]), q.rext[0], q.rmin[0]), fma_(mul((float)y, q.inv_res[1]), q.rext[1], q.rmin[1]),
	          fma_(mul((float)z, q.inv_res[2]), q.rext[2], q.rmin[2]));
}

// The network reads the warped grid point; the filter looks the running density grid up at the unwarped one (grid_samples_half_to_float
// with m_aabb).
template <bool ACC16>
__global__ void __launch_bounds__(128) k_density_on_grid(const DevModel m, const GridQuery q, const float* __restrict__ density_grid, float* __restrict__ out) {
	const uint32_t n = q.res[0] * q.res[1] * q.res[2];
	const uint32_t n_padded = ((n + 127u) / 128u) * 128u;  // the host checks that this fits 32 bits
	// the density MLP does not read the direction
	network_tiles<ACC16>(m, n, n_padded, true, v3(0.5f, 0.5f, 0.5f), [&](uint32_t i, V3& pw, V3&) {
		pw = warp_position(grid_point(q, i), q.tmin, q.tmax);
	}, [&](uint32_t i, bool valid, V3 pw, const uint32_t* dens, const uint32_t*) {
		if (!valid) return;
		float v = __half2float(__ushort_as_half((unsigned short)(dens[0] & 0xffffu)));  // the raw output, not the activated density
		const V3 p = unwarp_position(pw, q.tmin, q.tmax);
		const uint32_t mip = (uint32_t)mip_from_pos(p);
		if (__ldg(density_grid + cascaded_grid_idx_at(p, mip) + mip * GRIDVOL) < 0.01f) v = -10000.0f;  // NERF_MIN_OPTICAL_THICKNESS
		out[i] = v;
	});
}

// ---- marching cubes ------------------------------------------------------------------------------------------------
struct McGrid {
	const float* d;
	uint32_t rx, ry, rz, rxy;
	uint32_t n;  // rx * ry * rz
	float thresh;
};

// bit a set: the edge from grid point i along axis a (x, y, z) crosses the threshold (gen_vertices :225-263)
__device__ __forceinline__ uint32_t mc_cross_bits(const McGrid& g, uint32_t i, uint32_t x, uint32_t y, uint32_t z) {
	const bool in0 = __ldg(g.d + i) > g.thresh;
	uint32_t b = 0;
	if (x + 1 < g.rx && in0 != (__ldg(g.d + i + 1) > g.thresh)) b |= 1u;
	if (y + 1 < g.ry && in0 != (__ldg(g.d + i + g.rx) > g.thresh)) b |= 2u;
	if (z + 1 < g.rz && in0 != (__ldg(g.d + i + g.rxy) > g.thresh)) b |= 4u;
	return b;
}
// the configuration of the cell whose lowest corner is grid point i (gen_faces :600-618); 0 where no cell starts
__device__ __forceinline__ uint32_t mc_config(const McGrid& g, uint32_t i, uint32_t x, uint32_t y, uint32_t z) {
	if (x + 1 >= g.rx || y + 1 >= g.ry || z + 1 >= g.rz) return 0;
	const uint32_t o[8] = {0, 1, 1 + g.rx, g.rx, g.rxy, 1 + g.rxy, 1 + g.rx + g.rxy, g.rx + g.rxy};
	uint32_t c = 0;
#pragma unroll
	for (int k = 0; k < 8; ++k) c |= (__ldg(g.d + i + o[k]) > g.thresh ? 1u : 0u) << k;
	return c;
}
__device__ __forceinline__ void mc_coords(const McGrid& g, uint32_t i, uint32_t& x, uint32_t& y, uint32_t& z) {
	z = i / g.rxy;
	const uint32_t r = i - z * g.rxy;
	y = r / g.rx;
	x = r - y * g.rx;
}

// per CTA: the number of vertices owned by, and triangles of the cells starting at, its TILE grid points
__global__ void __launch_bounds__(THREADS) k_mc_count(const McGrid g, uint32_t* __restrict__ tile_nv, uint32_t* __restrict__ tile_nt) {
	using Reduce = cub::BlockReduce<uint32_t, THREADS>;
	__shared__ typename Reduce::TempStorage s_nv, s_nt;
	uint32_t nv = 0, nt = 0;
	const uint32_t first = blockIdx.x * TILE + threadIdx.x * PER_THREAD;
#pragma unroll
	for (uint32_t k = 0; k < PER_THREAD; ++k) {
		const uint32_t i = first + k;
		if (i >= g.n) break;
		uint32_t x, y, z;
		mc_coords(g, i, x, y, z);
		nv += __popc(mc_cross_bits(g, i, x, y, z));
		nt += kMcCount[mc_config(g, i, x, y, z)];
	}
	nv = Reduce(s_nv).Sum(nv);
	nt = Reduce(s_nt).Sum(nt);
	if (threadIdx.x == 0) { tile_nv[blockIdx.x] = nv; tile_nt[blockIdx.x] = nt; }
}

// exclusive scan of both tile arrays in place, in one CTA; totals[0], [1] = vertices, triangles (64-bit, so the host can reject
// meshes whose counts do not fit the 32-bit indices)
__global__ void __launch_bounds__(512) k_mc_scan(uint32_t n_tiles, uint32_t* __restrict__ tile_nv, uint32_t* __restrict__ tile_nt,
                                                  unsigned long long* __restrict__ totals) {
	using Scan = cub::BlockScan<unsigned long long, 512>;
	__shared__ typename Scan::TempStorage s;
	unsigned long long run_nv = 0, run_nt = 0;
	for (uint32_t base = 0; base < n_tiles; base += 512) {
		const uint32_t t = base + threadIdx.x;
		unsigned long long a = t < n_tiles ? tile_nv[t] : 0ull, b = t < n_tiles ? tile_nt[t] : 0ull, sa, sb;
		Scan(s).ExclusiveSum(a, a, sa);
		__syncthreads();
		Scan(s).ExclusiveSum(b, b, sb);
		__syncthreads();
		if (t < n_tiles) { tile_nv[t] = (uint32_t)(run_nv + a); tile_nt[t] = (uint32_t)(run_nt + b); }
		run_nv += sa;
		run_nt += sb;
	}
	if (threadIdx.x == 0) { totals[0] = run_nv; totals[1] = run_nt; }
}

// vertex ids (voff[i] = id of grid point i's first vertex) and positions, gen_vertices' arithmetic bit for bit:
// dt = (thresh - f0) / (f1 - f0) from the lower-index end, p = {x + dt, y, z} * scale + offset with the FMA nvcc contracts it to
__global__ void __launch_bounds__(THREADS) k_mc_vertices(const McGrid g, const uint32_t* __restrict__ tile_nv, float scx, float scy, float scz,
                                                         float ox, float oy, float oz, uint32_t* __restrict__ voff, float* __restrict__ verts) {
	using Scan = cub::BlockScan<uint32_t, THREADS>;
	__shared__ typename Scan::TempStorage s;
	const uint32_t first = blockIdx.x * TILE + threadIdx.x * PER_THREAD;
	uint32_t bits[PER_THREAD], cnt = 0;
#pragma unroll
	for (uint32_t k = 0; k < PER_THREAD; ++k) {
		const uint32_t i = first + k;
		bits[k] = 0;
		if (i < g.n) {
			uint32_t x, y, z;
			mc_coords(g, i, x, y, z);
			bits[k] = mc_cross_bits(g, i, x, y, z);
		}
		cnt += __popc(bits[k]);
	}
	uint32_t v;
	Scan(s).ExclusiveSum(cnt, v);
	v += tile_nv[blockIdx.x];
#pragma unroll
	for (uint32_t k = 0; k < PER_THREAD; ++k) {
		const uint32_t i = first + k;
		if (i >= g.n) break;
		voff[i] = v;
		if (!bits[k]) continue;
		uint32_t x, y, z;
		mc_coords(g, i, x, y, z);
		const float f0 = __ldg(g.d + i);
		const float fx = (float)x, fy = (float)y, fz = (float)z;
		const uint32_t step[3] = {1u, g.rx, g.rxy};
#pragma unroll
		for (uint32_t a = 0; a < 3; ++a) {
			if (!(bits[k] & (1u << a))) continue;
			const float f1 = __ldg(g.d + i + step[a]);
			const float dt = div_(sub(g.thresh, f0), sub(f1, f0));
			float* o = verts + 3 * (size_t)v;
			o[0] = fma_(a == 0 ? add(fx, dt) : fx, scx, ox);
			o[1] = fma_(a == 1 ? add(fy, dt) : fy, scy, oy);
			o[2] = fma_(a == 2 ? add(fz, dt) : fz, scz, oz);
			++v;
		}
	}
}

// the vertex id of cube edge e of the cell at grid point i: the edge's owner corner and axis (gen_faces :620-637), the owner's
// first vertex id from voff, plus the number of its crossing edges on lower axes (vertices are ordered x, y, z per grid point)
__device__ __forceinline__ uint32_t mc_edge_vertex(const McGrid& g, const uint32_t* __restrict__ voff, uint32_t i, uint32_t x, uint32_t y, uint32_t z, int e) {
	// owner corner (dx, dy, dz) and axis of edges 0..11
	const uint32_t code[12] = {0x000, 0x101, 0x020, 0x001, 0x040, 0x141, 0x060, 0x041, 0x002, 0x102, 0x122, 0x022};
	const uint32_t c = code[e];
	const uint32_t dx = (c >> 8) & 1u, dy = (c >> 5) & 1u, dz = (c >> 6) & 1u, axis = c & 3u;
	const uint32_t o = i + dx + dy * g.rx + dz * g.rxy;
	uint32_t v = __ldg(voff + o);
	if (axis > 0) {
		const uint32_t b = mc_cross_bits(g, o, x + dx, y + dy, z + dz);
		v += (b & 1u) + (axis > 1 ? ((b >> 1) & 1u) : 0u);
	}
	return v;
}

__global__ void __launch_bounds__(THREADS) k_mc_faces(const McGrid g, const uint32_t* __restrict__ tile_nt, const uint32_t* __restrict__ voff,
                                                      uint32_t* __restrict__ indices) {
	using Scan = cub::BlockScan<uint32_t, THREADS>;
	__shared__ typename Scan::TempStorage s;
	__shared__ int8_t s_tri[256][NSB_MC_ROW];
	for (uint32_t k = threadIdx.x; k < 256 * NSB_MC_ROW; k += THREADS) (&s_tri[0][0])[k] = (&kMcTri[0][0])[k];
	__syncthreads();
	const uint32_t first = blockIdx.x * TILE + threadIdx.x * PER_THREAD;
	uint32_t cfg[PER_THREAD], cnt = 0;
#pragma unroll
	for (uint32_t k = 0; k < PER_THREAD; ++k) {
		const uint32_t i = first + k;
		cfg[k] = 0;
		if (i < g.n) {
			uint32_t x, y, z;
			mc_coords(g, i, x, y, z);
			cfg[k] = mc_config(g, i, x, y, z);
		}
		cnt += kMcCount[cfg[k]];
	}
	uint32_t t;
	Scan(s).ExclusiveSum(cnt, t);
	t += tile_nt[blockIdx.x];
#pragma unroll
	for (uint32_t k = 0; k < PER_THREAD; ++k) {
		if (!cfg[k]) continue;
		const uint32_t i = first + k;
		uint32_t x, y, z;
		mc_coords(g, i, x, y, z);
		const int8_t* row = s_tri[cfg[k]];
		for (int j = 0; j < NSB_MC_ROW && row[j] >= 0; ++j) indices[3 * (size_t)t + j] = mc_edge_vertex(g, voff, i, x, y, z, row[j]);
		t += kMcCount[cfg[k]];
	}
}

// ---- vertex normals: per-vertex triangle lists (CSR), then a sum in ascending triangle order --------------------------
__global__ void k_mesh_degree(uint32_t n_tris, const uint32_t* __restrict__ indices, uint32_t* __restrict__ deg) {
	const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= n_tris) return;
	for (int k = 0; k < 3; ++k) atomicAdd(deg + indices[3 * (size_t)t + k], 1u);  // integer counts: the result does not depend on the order
}
__global__ void k_mesh_fill(uint32_t n_tris, const uint32_t* __restrict__ indices, const uint32_t* __restrict__ start, uint32_t* __restrict__ cursor,
                            uint32_t* __restrict__ adj) {
	const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= n_tris) return;
	for (int k = 0; k < 3; ++k) {
		const uint32_t v = indices[3 * (size_t)t + k];
		adj[start[v] + atomicAdd(cursor + v, 1u)] = t;  // the slot order varies; k_mesh_normals visits the list sorted
	}
}
// normal = sum over the vertex's triangles, in ascending triangle index, of (pb - pa) x (pa - pc) (accumulate_1ring :293);
// rows n_vertices .. n_rows - 1 are the reference's padding and get a zero normal
__global__ void k_mesh_normals(uint32_t n_vertices, uint32_t n_rows, const float* __restrict__ verts, const uint32_t* __restrict__ indices,
                               const uint32_t* __restrict__ start, const uint32_t* __restrict__ adj, float* __restrict__ normals) {
	const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
	if (v >= n_rows) return;
	V3 n = v3(0.0f, 0.0f, 0.0f);
	if (v < n_vertices) {
		const uint32_t b = start[v], e = start[v + 1];
		uint32_t last = 0;
		for (uint32_t k = b; k < e; ++k) {  // selection of the next larger triangle index: lists are a few entries long
			uint32_t t = 0xffffffffu;
			for (uint32_t j = b; j < e; ++j) {
				const uint32_t a = adj[j];
				if ((k == b || a > last) && a < t) t = a;
			}
			last = t;
			const V3 pa = ldv(verts, indices[3 * (size_t)t]), pb = ldv(verts, indices[3 * (size_t)t + 1]), pc = ldv(verts, indices[3 * (size_t)t + 2]);
			n = vadd(n, cross3(vsub(pb, pa), vsub(pa, pc)));
		}
	}
	normals[3 * (size_t)v] = n.x;
	normals[3 * (size_t)v + 1] = n.y;
	normals[3 * (size_t)v + 2] = n.z;
}

struct Aabb { float mn[3], mx[3]; };

// ---- vertex colours ------------------------------------------------------------------------------------------------
// dir = normalize(pos - 0.5) (Eigen normalized(): unchanged when the norm is 0), the network at {warp(pos), warp(dir)}, then
// network_to_rgb and, for linear colours, linear_to_srgb; every row including the padding (whose position is the origin), so n_rows
// (a multiple of 128) rows are all valid
template <bool ACC16>
__global__ void __launch_bounds__(128) k_mesh_colors(const DevModel m, uint32_t n_rows, const float* __restrict__ verts, const Aabb train,
                                                     int rgb_activation, int linear_colors, float* __restrict__ colors) {
	network_tiles<ACC16>(m, n_rows, n_rows, false, v3(0.5f, 0.5f, 0.5f), [&](uint32_t i, V3& pw, V3& dw) {
		const V3 p = ldv(verts, i);
		V3 d = vsub(p, v3(0.5f, 0.5f, 0.5f));
		const float n2 = dot3(d, d);
		if (n2 > 0.0f) { const float nn = __fsqrt_rn(n2); d = v3(div_(d.x, nn), div_(d.y, nn), div_(d.z, nn)); }
		pw = warp_position(p, train.mn, train.mx);
		dw = warp_direction(d);
	}, [&](uint32_t i, bool, V3, const uint32_t*, const uint32_t* rgbo) {
		const unsigned short h[3] = {(unsigned short)(rgbo[0] & 0xffffu), (unsigned short)(rgbo[0] >> 16), (unsigned short)(rgbo[1] & 0xffffu)};
#pragma unroll
		for (int k = 0; k < 3; ++k) {
			float c = network_to_rgb(__half2float(__ushort_as_half(h[k])), rgb_activation);
			if (linear_colors) c = linear_to_srgb(c);
			colors[3 * (size_t)i + k] = c;
		}
	});
}

}  // namespace mesh
