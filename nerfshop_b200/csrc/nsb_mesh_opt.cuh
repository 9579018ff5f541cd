// Mesh optimisation on the device: the kernels behind nsb_density_gradient and nsb_mesh_optimise.
// Included by nsb_kernels.cu after nsb_mesh.cuh (encode_to_a32, the tc:: layer chain, mesh::Aabb).
//
//   k_density_gradient  NerfNetwork::density + NerfNetwork::input_gradient(3) (nerf_network_full.h:142-221, 223-239) in one pass:
//                       hash grid -> L1 -> L2 on wgmma (the raw density, bit for bit nsb_density's), then the backward of the density MLP
//                       seeded with 128 at output 0 (tcnn's backprop_scale), and the hash grid's position derivative; DESIGN §7.2
//   k_mesh_opt_step     compute_mesh_1ring (marching_cubes.cu:267-302, 656-662) + compute_mesh_opt_gradients_kernel (:664-696) + tcnn Adam
//                       for non-matrix parameters, one thread per vertex row; positions ping-pong between two buffers
namespace meshopt {

constexpr uint32_t WT_BYTES = 32 * 64 * 2;  // W1^T [32 x 64], the B operand of the first layer's backward

// The one-tile layout of the network kernels plus the W1^T operand this kernel stages for itself
struct __align__(128) GradSmem {
	tc::TileSmem t;
	uint8_t wt[WT_BYTES];
};

struct GradIo {
	const float* in;      // VERTS: vertex rows (3 floats, world units, warped with `train`); else NerfCoordinate rows (7 floats, warped)
	uint32_t n;           // rows to read
	uint32_t n_padded;    // rows of the fp16 outputs (a multiple of 128)
	float* grad;          // 3 floats of row i at grad + i * grad_stride; may alias `in` (one thread reads and writes its own row)
	uint32_t grad_stride;
	__half* dens;         // [n_padded] raw density, may be null
	__half* dfeat;        // [32 x n_padded] dL/dfeatures scaled by 128, may be null
	mesh::Aabb train;
};

// dL/dpos of level l: sum over k = 2l+f ascending of fma(float(dfeat_k), dy_dx[k][d], acc), dy_dx[k][d] = the sum over the four corner pairs
// along d (other dims in ascending order, bit 0 = the lower one) of fma(weight, float(v_right) - float(v_left), .), weight = scale * w_o0 * w_o1
template <int MODE>
__device__ __forceinline__ void grid_backward_level(const DevLevel& L, float x, float y, float z, uint32_t df_bits, float* g) {
	const float px = fma_(L.scale, x, 0.5f), py = fma_(L.scale, y, 0.5f), pz = fma_(L.scale, z, 0.5f);
	const float fx = floorf(px), fy = floorf(py), fz = floorf(pz);
	const float w[3] = {sub(px, fx), sub(py, fy), sub(pz, fz)};
	const uint32_t gx = (uint32_t)(int)fx, gy = (uint32_t)(int)fy, gz = (uint32_t)(int)fz;
	float2 v[8];
#pragma unroll
	for (int c = 0; c < 8; ++c) v[c] = __half22float2(__ldg(L.base + grid_index<MODE>(L, gx + (c & 1), gy + ((c >> 1) & 1), gz + ((c >> 2) & 1))));
	const float df0 = h_lo(df_bits), df1 = h_hi(df_bits);
#pragma unroll
	for (int d = 0; d < 3; ++d) {
		const int o0 = d == 0 ? 1 : 0, o1 = d == 2 ? 1 : 2;
		float s0 = 0.0f, s1 = 0.0f;
#pragma unroll
		for (int idx = 0; idx < 4; ++idx) {
			const float weight = mul(mul(L.scale, (idx & 1) ? w[o0] : sub(1.0f, w[o0])), (idx & 2) ? w[o1] : sub(1.0f, w[o1]));
			const int cl = ((idx & 1) << o0) | (((idx >> 1) & 1) << o1), cr = cl | (1 << d);
			s0 = fma_(weight, sub(v[cr].x, v[cl].x), s0);
			s1 = fma_(weight, sub(v[cr].y, v[cl].y), s1);
		}
		g[d] = fma_(df1, s1, fma_(df0, s0, g[d]));
	}
}

template <bool ACC16, bool VERTS>
__global__ void __launch_bounds__(128) k_density_gradient(const DevModel m, const GradIo io) {
	extern __shared__ __align__(128) uint8_t smem_raw[];
	GradSmem& S = *reinterpret_cast<GradSmem*>(smem_raw);
	const uint32_t tid = threadIdx.x, lane = tid & 31u;
	tc::tile_setup(S.t, m.w_image);
	// W1^T from the staged W1 image: element (n = feature f, k = hidden j) of the [32 x 64] operand <- W1 (n = j, k = f)
	for (uint32_t e = tid; e < 32 * 64; e += 128) {
		const uint32_t f = e & 31u, j = e >> 5;
		const uint16_t h = *reinterpret_cast<const uint16_t*>(S.t.w + tc::W1_OFF + (f / 8) * (64 * 16) + j * 16 + (f % 8) * 2);
		*reinterpret_cast<uint16_t*>(S.wt + (j / 8) * (32 * 16) + f * 16 + (j % 8) * 2) = h;
	}
	tc::fence_async_smem();
	__syncthreads();
	const uint32_t a32 = tc::smem_u32(S.t.a32), w = tc::smem_u32(S.t.w), wt = tc::smem_u32(S.wt);
	const __half2 g_scale = __floats2half2_rn(128.0f, 128.0f), zero = __floats2half2_rn(0.0f, 0.0f);
	// tile indices, as network_tiles walks them (a row base would wrap past 2^32 for n_padded near it)
	const uint32_t n_tiles = (uint32_t)(((uint64_t)io.n_padded + 127u) / 128u);
	for (uint32_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
		const uint32_t i = t * 128u + tid;
		const bool valid = i < io.n;
		V3 pw = v3(0, 0, 0);
		if (valid) pw = VERTS ? warp_position(ldv(io.in, i), io.train.mn, io.train.mx) : v3(io.in[7 * (size_t)i], io.in[7 * (size_t)i + 1], io.in[7 * (size_t)i + 2]);
		encode_to_a32(S.t.a32, m, valid, pw, tid);
		tc::fence_async_smem();
		__syncthreads();  // every sample's grid features are in place
#pragma unroll 1
		for (uint32_t h = 0; h < 2; ++h) {
			tc::Acc<64, ACC16> x;
			tc::Acc<16, ACC16> o;
			tc::Acc<32, ACC16> gd;
			tc::layer_ss<64, 32, ACC16>(x.r, a32 + h * 64 * 16, w + tc::W1_OFF);  // L1, as tc::run_network
			tc::layer_rs<16, 64, ACC16>(o.r, x.r, w + tc::W2_OFF);                // L2
			tc::store_out16<ACC16>(S.t.a32, 6, tid, h, o.r);
			// dL/dh = relu'(h) * 128 * W2[0, :]: pair p of the L1 accumulator covers columns 8*(p/2) + 2*(lane%4) + {0,1}, which is the A
			// fragment of k-step p/4 (as in tc::layer_rs); the mask reads the fp16-rounded activation
			uint32_t a[4][4];
#pragma unroll
			for (int k = 0; k < 4; ++k)
#pragma unroll
				for (int q = 0; q < 4; ++q) {
					const int p = 4 * k + q;
					const uint32_t col = 8u * (uint32_t)(p >> 1) + 2u * (lane & 3u);
					const __half2 w2 = *reinterpret_cast<const __half2*>(S.t.w + tc::W2_OFF + (col / 8) * (16 * 16) + (col % 8) * 2);
					uint32_t hp = tc::acc_pair<ACC16>(x.r, p);
					a[k][q] = tc::pack_h2(__hmul2(__hmul2(w2, g_scale), __hgt2(*reinterpret_cast<__half2*>(&hp), zero)));
				}
			tc::wg_fence();
#pragma unroll
			for (uint32_t k = 0; k < 4; ++k) tc::wgmma_rs<32, ACC16>(gd.r, a[k], tc::make_desc(wt + k * 2 * (32 * 16), 32 * 16, 128), k > 0 ? 1u : 0u);
			tc::wg_commit();
			tc::wg_wait();
			tc::reg_fence<tc::Acc<32, ACC16>::R>(gd.r);
			// dfeat -> this half's rows of chunks 0-3 (their first-layer operand, which L1 has finished reading)
			tc::store_out16<ACC16>(S.t.a32, 0, tid, h, gd.r);
			tc::store_out16<ACC16>(S.t.a32, 2, tid, h, gd.r + (ACC16 ? 4 : 8));
		}
		__syncwarp();
		const uint32_t dens_bits = tc::load_chunk(S.t.a32, 6, tid).x;
		if (i < io.n_padded) {
			if (io.dens) io.dens[i] = __ushort_as_half((unsigned short)(dens_bits & 0xffffu));
			if (io.dfeat) {
#pragma unroll
				for (uint32_t c = 0; c < 4; ++c) {
					const uint4 u = tc::load_chunk(S.t.a32, c, tid);
					const uint32_t r[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
					for (int k = 0; k < 4; ++k) {
						io.dfeat[(size_t)(8 * c + 2 * k) * io.n_padded + i] = __ushort_as_half((unsigned short)(r[k] & 0xffffu));
						io.dfeat[(size_t)(8 * c + 2 * k + 1) * io.n_padded + i] = __ushort_as_half((unsigned short)(r[k] >> 16));
					}
				}
			}
		}
		if (valid) {
			float g[3] = {0.0f, 0.0f, 0.0f};
			const uint8_t* row = S.t.a32 + tc::phys_row(tid) * 16;
#pragma unroll 1
			for (uint32_t l = 0; l < MAX_LEVELS; ++l) {
				const uint32_t df = *reinterpret_cast<const uint32_t*>(row + (l >> 2) * (tc::ROWS * 16) + (l & 3u) * 4);  // features 2l, 2l+1
				grid_backward_level<2>(m.levels[l], pw.x, pw.y, pw.z, df, g);
			}
			float* o = io.grad + (size_t)i * io.grad_stride;
			o[0] = mul(g[0], 0.0078125f);  // 1 / backprop_scale
			o[1] = mul(g[1], 0.0078125f);
			o[2] = mul(g[2], 0.0078125f);
		}
		__syncthreads();  // the tile is done with the operand space
	}
}

struct OptParams {
	float thresh, k_smooth, k_density, k_inflate;
};
// tcnn Adam of Testbed::marching_cubes (testbed_nerf.cu:4636-4643): learning rate 1e-4, beta1 0.9, beta2 0.99, epsilon 1e-8
constexpr float ADAM_LR = 1e-4f, ADAM_B1 = 0.9f, ADAM_B2 = 0.99f, ADAM_EPS = 1e-8f;

__device__ __forceinline__ V3 normalized(V3 v) {  // Eigen normalized(): unchanged when the norm is 0
	const float n2 = dot3(v, v);
	if (!(n2 > 0.0f)) return v;
	const float n = __fsqrt_rn(n2);
	return v3(div_(v.x, n), div_(v.y, n), div_(v.z, n));
}

// One row: the 1-ring sum and normal of pos_in (triangles in ascending index, like k_mesh_normals), the opt gradient, then Adam per coordinate
// into pos_out. Rows n_vertices .. n_rows - 1 are the padding: no triangles, so their centroid is the origin and their normal zero.
__global__ void k_mesh_opt_step(uint32_t n_vertices, uint32_t n_rows, const float* __restrict__ pos_in, float* __restrict__ pos_out,
                                const uint32_t* __restrict__ indices, const uint32_t* __restrict__ start, const uint32_t* __restrict__ adj,
                                const __half* __restrict__ dens, const float* __restrict__ grad, const OptParams p, float* __restrict__ m1,
                                float* __restrict__ m2, uint32_t* __restrict__ steps, float* __restrict__ normals) {
	const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
	if (v >= n_rows) return;
	V3 s = v3(0.0f, 0.0f, 0.0f), nrm = v3(0.0f, 0.0f, 0.0f);
	float wsum = 0.0f;
	if (v < n_vertices) {
		const uint32_t b = start[v], e = start[v + 1];
		uint32_t last = 0;
		for (uint32_t k = b; k < e; ++k) {
			uint32_t t = 0xffffffffu;
			for (uint32_t j = b; j < e; ++j) {
				const uint32_t a = adj[j];
				if ((k == b || a > last) && a < t) t = a;
			}
			last = t;
			const uint32_t ia = indices[3 * (size_t)t], ib = indices[3 * (size_t)t + 1], ic = indices[3 * (size_t)t + 2];
			const V3 pa = ldv(pos_in, ia), pb = ldv(pos_in, ib), pc = ldv(pos_in, ic);
			// accumulate_1ring: a gets pb + pc, b gets pa + pc, c gets pb + pa, each with weight 2
			s = vadd(s, ia == v ? vadd(pb, pc) : (ib == v ? vadd(pa, pc) : vadd(pb, pa)));
			wsum = add(wsum, 2.0f);
			nrm = vadd(nrm, cross3(vsub(pb, pa), vsub(pa, pc)));
		}
	}
	normals[3 * (size_t)v] = nrm.x;
	normals[3 * (size_t)v + 1] = nrm.y;
	normals[3 * (size_t)v + 2] = nrm.z;
	// compute_mesh_opt_gradients_kernel
	if (wsum <= 0.0f) wsum = 1.0f;
	const float inv = div_(1.0f, wsum);
	const V3 src = ldv(pos_in, v);
	// src - p.head<3>() * (1/w): nvcc contracts the product into the subtraction (read off the SASS of the reference's kernel)
	const V3 sg = v3(fma_(-inv, s.x, src.x), fma_(-inv, s.y, src.y), fma_(-inv, s.z, src.z));
	const V3 n = normalized(ldv(grad, v));
	const V3 nn = normalized(nrm);
	const float sgn = copysignf(1.0f, sub(__half2float(dens[v]), p.thresh));
	// n*sign*k_density + sg*k_smooth - nn*k_inflate, contracted as the reference's kernel compiles: fma(n*sign, k_density, sg*k_smooth), then
	// fma(-nn, k_inflate, .)
	const float gv[3] = {fma_(-nn.x, p.k_inflate, fma_(mul(n.x, sgn), p.k_density, mul(sg.x, p.k_smooth))),
	                     fma_(-nn.y, p.k_inflate, fma_(mul(n.y, sgn), p.k_density, mul(sg.y, p.k_smooth))),
	                     fma_(-nn.z, p.k_inflate, fma_(mul(n.z, sgn), p.k_density, mul(sg.z, p.k_smooth)))};
	const float pv[3] = {src.x, src.y, src.z};
#pragma unroll
	for (int c = 0; c < 3; ++c) {
		const size_t j = 3 * (size_t)v + c;
		float x = pv[c];
		const float g = gv[c];
		if (g != 0.0f) {  // a non-matrix parameter with a zero gradient is skipped: no moment update, no step
			const float mm = fma_(ADAM_B1, m1[j], mul(sub(1.0f, ADAM_B1), g));
			const float vv = fma_(ADAM_B2, m2[j], mul(sub(1.0f, ADAM_B2), mul(g, g)));
			m1[j] = mm;
			m2[j] = vv;
			const uint32_t t = steps[j] + 1u;
			steps[j] = t;
			const float lr = mul(ADAM_LR, div_(__fsqrt_rn(sub(1.0f, powf(ADAM_B2, (float)t))), sub(1.0f, powf(ADAM_B1, (float)t))));
			// tcnn adam_step: effective_learning_rate = lr_t / (sqrtf(v) + epsilon), new = weight - effective_learning_rate * m
			const float eff = div_(lr, add(__fsqrt_rn(vv), ADAM_EPS));
			x = fma_(-eff, mm, x);
		}
		pos_out[j] = x;
	}
}

}  // namespace meshopt
