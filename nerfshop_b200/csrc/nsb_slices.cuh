// Density and RGBA slices on the device: the kernels behind nsb_rgba_on_grid, nsb_density_png and nsb_rgba_png.
// Included by nsb_kernels.cu after nsb_mesh.cuh (mesh::GridQuery, mesh::grid_point, network_tiles).
//
//   k_rgba_on_grid   Testbed::get_rgba_on_grid (testbed_nerf.cu:4588-4612): generate_grid_samples_nerf_uniform_dir (:416-427)
//                    + NerfNetwork::inference + compute_nerf_density (:624-635) in one pass, no position buffer, no 1M batches
//   k_density_png    save_density_grid_to_png (marching_cubes.cu:898-974): the 8-bit mosaic of the z slices and both counts
//   k_rgba_png       save_rgba_grid_to_png_sequence (marching_cubes.cu:979-1015): one RGBA image per z slice, back to back
namespace slices {

// ---- RGBA on a grid ------------------------------------------------------------------------------------------------
// The positions are mesh::grid_point's: the PTX of the reference's generate_grid_samples_nerf_uniform_dir contracts
// x * (1/res) * (max - min) + min into mul + fma like its uniform variant. One direction for the whole launch.
// The network output rows 0-3 (rgb, then the density via extract_density) become float as tcnn's float inference output does;
// then compute_nerf_density: a = clamp(1 - __expf(-network_to_density(d) / 100), 0, 1) with div.rn, rgb = network_to_rgb(c) * a.
template <bool ACC16>
__global__ void __launch_bounds__(128) k_rgba_on_grid(const DevModel m, const mesh::GridQuery q, float dx, float dy, float dz, int rgb_act, int density_act,
                                                      float4* __restrict__ out) {
	const uint32_t n = q.res[0] * q.res[1] * q.res[2];
	const uint32_t n_padded = ((n + 127u) / 128u) * 128u;  // the host checks that this fits 32 bits
	network_tiles<ACC16>(m, n, n_padded, false, warp_direction(v3(dx, dy, dz)), [&](uint32_t i, V3& pw, V3&) {
		pw = warp_position(mesh::grid_point(q, i), q.tmin, q.tmax);
	}, [&](uint32_t i, bool valid, V3, const uint32_t* dens, const uint32_t* rgbo) {
		if (!valid) return;
		const float d = __half2float(__ushort_as_half((unsigned short)(dens[0] & 0xffffu)));
		const float a = clampf(sub(1.0f, __expf(div_(-network_to_density(d, density_act), 100.0f))), 0.0f, 1.0f);
		const unsigned short h[3] = {(unsigned short)(rgbo[0] & 0xffffu), (unsigned short)(rgbo[0] >> 16), (unsigned short)(rgbo[1] & 0xffffu)};
		float c[3];
#pragma unroll
		for (int k = 0; k < 3; ++k) c[k] = mul(network_to_rgb(__half2float(__ushort_as_half(h[k])), rgb_act), a);
		out[i] = make_float4(c[0], c[1], c[2], a);
	});
}

// ---- slice images --------------------------------------------------------------------------------------------------
// res: the grid as stored (x fastest). After the optional y/z swap the images have rows of res_x pixels, res_y' = res_z rows and
// res_z' = res_y slices; without the swap the rows run from y = res_y - 1 down to 0. src_index gives the grid point of pixel (x, y) of
// slice z in those swapped coordinates (the two index expressions of marching_cubes.cu:955-957 and :999).
struct Slices {
	uint32_t rx, ry, rz;  // the grid
	uint32_t sy, sz;      // image rows and slice count after the swap
	uint32_t swap;
};
__device__ __forceinline__ uint64_t src_index(const Slices& s, uint32_t x, uint32_t y, uint32_t z) {
	const uint64_t rxy = (uint64_t)s.rx * s.ry;
	return s.swap ? x + (uint64_t)z * s.rx + (uint64_t)y * rxy : x + (uint64_t)(s.ry - 1 - y) * s.rx + (uint64_t)z * rxy;
}
// (uint8_t)tcnn::clamp(v, 0.f, 255.f): truncation toward zero (NaN gives 0, as x86's cvttss2si does in the low byte)
__device__ __forceinline__ uint8_t to_u8(float v) { return (uint8_t)__float2uint_rz(clampf(v, 0.0f, 255.0f)); }

// One thread per mosaic pixel (u, v): grid point (u % res_x, v % res_y', u / res_x + (v / res_y') * nacross), 0 past the last slice;
// the value is (d - thresh) * (128 / range) + 128.5 with the product and the sum rounded separately, as the reference's host loop.
// Thread i < n_points also counts, at the interior grid point i (1 <= x, y, z <= res - 2, marching_cubes.cu:906-935), the cell whose
// corners are not all on one side of thresh and the lattice point with a 6-neighbour on the other side; warp sums, then one 64-bit
// integer atomic per warp: the counts do not depend on the order.
__global__ void __launch_bounds__(256) k_density_png(const Slices s, const float* __restrict__ d, float thresh, float scale, uint32_t w, uint32_t nacross,
                                                      uint8_t* __restrict__ pixels, unsigned long long* __restrict__ counts) {
	const uint64_t n_px = (uint64_t)w * (s.sy * (uint64_t)((s.sz + nacross - 1) / nacross));
	const uint64_t n_pts = (uint64_t)s.rx * s.ry * s.rz;
	const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
	const uint64_t end = ((n_px > n_pts ? n_px : n_pts) + 31) & ~31ull;  // whole warps stay in the loop for the warp sums
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < end; i += stride) {
		if (i < n_px) {
			const uint32_t u = (uint32_t)(i % w), v = (uint32_t)(i / w);
			const uint32_t x = u % s.rx, y = v % s.sy, z = u / s.rx + (v / s.sy) * nacross;
			pixels[i] = z < s.sz ? to_u8(add(mul(sub(__ldg(d + src_index(s, x, y, z)), thresh), scale), 128.5f)) : (uint8_t)0;
		}
		uint32_t voxel = 0, near = 0;
		if (i < n_pts) {
			const uint64_t rxy = (uint64_t)s.rx * s.ry;
			const uint32_t z = (uint32_t)(i / rxy), r = (uint32_t)(i - z * rxy), y = r / s.rx, x = r - y * s.rx;
			if (x >= 1 && y >= 1 && z >= 1 && x + 1 < s.rx && y + 1 < s.ry && z + 1 < s.rz) {
				const uint64_t ox = 1, oy = s.rx, oz = rxy;
				const bool in0 = __ldg(d + i) < thresh;
				uint32_t cnt = 0;
#pragma unroll
				for (int k = 0; k < 8; ++k) cnt += __ldg(d + i + ((k & 1) ? ox : 0) + ((k & 2) ? oy : 0) + ((k & 4) ? oz : 0)) < thresh;
				voxel = cnt > 0 && cnt < 8;
				near = ((__ldg(d + i + ox) < thresh) != in0) | ((__ldg(d + i - ox) < thresh) != in0) | ((__ldg(d + i + oy) < thresh) != in0) |
				       ((__ldg(d + i - oy) < thresh) != in0) | ((__ldg(d + i + oz) < thresh) != in0) | ((__ldg(d + i - oz) < thresh) != in0);
			}
		}
		voxel = __reduce_add_sync(0xffffffffu, voxel);
		near = __reduce_add_sync(0xffffffffu, near);
		if ((threadIdx.x & 31u) == 0) {
			if (voxel) atomicAdd(counts, (unsigned long long)voxel);
			if (near) atomicAdd(counts + 1, (unsigned long long)near);
		}
	}
}

// One thread per pixel of all slices: slice z of res_x x res_y' pixels at byte z * res_x * res_y' * 4; (uint8_t)clamp(v * 255, 0, 255) per channel
__global__ void __launch_bounds__(256) k_rgba_png(const Slices s, const float4* __restrict__ rgba, uchar4* __restrict__ pixels) {
	const uint64_t per_slice = (uint64_t)s.rx * s.sy, n = per_slice * s.sz;
	for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
		const uint32_t z = (uint32_t)(i / per_slice), r = (uint32_t)(i - z * per_slice), y = r / s.rx, x = r - y * s.rx;
		const float4 c = __ldg(rgba + src_index(s, x, y, z));
		pixels[i] = make_uchar4(to_u8(mul(c.x, 255.0f)), to_u8(mul(c.y, 255.0f)), to_u8(mul(c.z, 255.0f)), to_u8(mul(c.w, 255.0f)));
	}
}

}  // namespace slices
