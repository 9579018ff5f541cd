/*
 * mesh_opt_oracle.cpp — CPU restatement of the density input gradient (NerfNetwork::input_gradient(3)) and of one step of
 * Testbed::optimise_mesh_step. TEST INFRASTRUCTURE ONLY, like nerfshop_oracle.cpp, whose model, hash grid and MLP restatement it
 * reuses (it is compiled into the same library; oracle/mesh_opt_oracle.py builds it).
 *
 * Numerics contract as nerfshop_oracle.cpp: fp32 ops as written, FMA only where fmaf() is spelled out (compile with -ffp-contract=off).
 * The tiny-cuda-nn parts (backward of the fully fused MLP, grid input gradient, Adam) are a restatement of the published algorithm of that
 * era [tcnn-ext] (SURVEY.md Appendix B): the submodule is absent, so they are not verified against its code.
 */
#include "nerfshop_oracle.cpp"

namespace {

// tcnn kernel_grid with prepare_input_gradients (linear interpolation) + kernel_grid_backward_input: dL/dx[d] = the fp32 chain
// fmaf(float(dfeat_k), dy_dx[k][d], acc) over k = 2l + f ascending, dy_dx[k][d] = the chain over the four corner pairs along d (the other
// two dims ascending, bit 0 = the lower one) of fmaf(weight, float(v_right) - float(v_left), acc), weight = scale * w_o0 * w_o1; times 1/128.
void grid_backward(const Model& m, const float* x, const uint16_t* dfeat, float* out) {
	float g[3] = {0.0f, 0.0f, 0.0f};
	for (uint32_t l = 0; l < m.desc.n_levels; ++l) {
		const Level& L = m.levels[l];
		float w[3];
		uint32_t gp[3];
		for (int dim = 0; dim < 3; ++dim) {
			float p = fmaf(L.scale, x[dim], 0.5f);
			float fl = floorf(p);
			gp[dim] = (uint32_t)cvt_rzi_s32(fl);
			w[dim] = p - fl;
		}
		for (int d = 0; d < 3; ++d) {
			const int o0 = d == 0 ? 1 : 0, o1 = d == 2 ? 1 : 2;
			float s[2] = {0.0f, 0.0f};
			for (int idx = 0; idx < 4; ++idx) {
				const float weight = (L.scale * ((idx & 1) ? w[o0] : 1.0f - w[o0])) * ((idx & 2) ? w[o1] : 1.0f - w[o1]);
				uint32_t gl[3];
				gl[o0] = gp[o0] + (uint32_t)(idx & 1);
				gl[o1] = gp[o1] + (uint32_t)((idx >> 1) & 1);
				gl[d] = gp[d];
				const uint16_t* vl = m.grid + ((uint64_t)L.offset + grid_entry(L, gl)) * 2;
				gl[d] = gp[d] + 1u;
				const uint16_t* vr = m.grid + ((uint64_t)L.offset + grid_entry(L, gl)) * 2;
				for (int f = 0; f < 2; ++f) s[f] = fmaf(weight, h2f(vr[f]) - h2f(vl[f]), s[f]);
			}
			for (int f = 0; f < 2; ++f) g[d] = fmaf(h2f(dfeat[2 * l + f]), s[f], g[d]);
		}
	}
	for (int d = 0; d < 3; ++d) out[d] = g[d] * 0.0078125f;
}

// The density MLP forward (nerfshop_oracle.cpp's network_forward, density only) and its backward seeded with 128 at output 0: g = 128 * W2[0, :]
// (exact in fp16), masked by the fp16 activation h > 0, then dfeat = W1^T g through mlp_layer, i.e. under the same accumulator policy.
void density_backward(const Model& m, V3 pos_w, uint16_t* dens, uint16_t* dfeat) {
	uint16_t feat[32], h1[64], dout[16], g[64];
	encode_grid(m, pos_w, feat);
	mlp_layer(m.wf[0].data(), 64, 32, feat, true, h1);
	mlp_layer(m.wf[1].data(), 16, 64, h1, false, dout);
	*dens = dout[0];
	for (int j = 0; j < 64; ++j) g[j] = h2f(h1[j]) > 0.0f ? f2h(128.0f * m.wf[1][j]) : (uint16_t)0;
	float w1t[32 * 64];
	for (int f = 0; f < 32; ++f)
		for (int j = 0; j < 64; ++j) w1t[f * 64 + j] = m.wf[0][j * 32 + f];
	mlp_layer(w1t, 32, 64, g, false, dfeat);
}

// ---- float64 restatement without rounding, for the finite-difference check of the chain rule ----
double density_f64(const Model& m, const double* x, double* grad /* may be null */) {
	double feat[32], dy_dx[32][3];
	for (uint32_t l = 0; l < m.desc.n_levels; ++l) {
		const Level& L = m.levels[l];
		double w[3];
		uint32_t gp[3];
		for (int dim = 0; dim < 3; ++dim) {
			double p = (double)L.scale * x[dim] + 0.5;
			double fl = std::floor(p);
			gp[dim] = (uint32_t)cvt_rzi_s32(fl);  // the float64 floor converted as the device converts its float floor
			w[dim] = p - fl;
		}
		feat[2 * l] = feat[2 * l + 1] = 0.0;
		for (int d = 0; d < 3; ++d) dy_dx[2 * l][d] = dy_dx[2 * l + 1][d] = 0.0;
		for (uint32_t c = 0; c < 8; ++c) {
			uint32_t gl[3];
			double wt = 1.0, dw[3];
			for (int dim = 0; dim < 3; ++dim) gl[dim] = gp[dim] + ((c >> dim) & 1u);
			for (int dim = 0; dim < 3; ++dim) wt *= ((c >> dim) & 1u) ? w[dim] : 1.0 - w[dim];
			for (int d = 0; d < 3; ++d) {  // d weight / d x_d = scale * (+-1) * product of the other two
				dw[d] = (double)L.scale * (((c >> d) & 1u) ? 1.0 : -1.0);
				for (int o = 0; o < 3; ++o)
					if (o != d) dw[d] *= ((c >> o) & 1u) ? w[o] : 1.0 - w[o];
			}
			const uint16_t* e = m.grid + ((uint64_t)L.offset + grid_entry(L, gl)) * 2;
			for (int f = 0; f < 2; ++f) {
				feat[2 * l + f] += wt * h2f(e[f]);
				for (int d = 0; d < 3; ++d) dy_dx[2 * l + f][d] += dw[d] * h2f(e[f]);
			}
		}
	}
	double h[64], dens = 0.0;
	for (int j = 0; j < 64; ++j) {
		double a = 0.0;
		for (int k = 0; k < 32; ++k) a += (double)m.wf[0][j * 32 + k] * feat[k];
		h[j] = a > 0.0 ? a : 0.0;
		dens += (double)m.wf[1][j] * h[j];
	}
	if (grad) {
		double dfeat[32];
		for (int k = 0; k < 32; ++k) {
			dfeat[k] = 0.0;
			for (int j = 0; j < 64; ++j)
				if (h[j] > 0.0) dfeat[k] += 128.0 * (double)m.wf[1][j] * (double)m.wf[0][j * 32 + k];
		}
		for (int d = 0; d < 3; ++d) {
			grad[d] = 0.0;
			for (int k = 0; k < 32; ++k) grad[d] += dfeat[k] * dy_dx[k][d];
			grad[d] /= 128.0;
		}
	}
	return dens;
}

inline V3 sub3(V3 a, V3 b) { return v3(a.x - b.x, a.y - b.y, a.z - b.z); }
inline V3 add3(V3 a, V3 b) { return v3(a.x + b.x, a.y + b.y, a.z + b.z); }
// the contracted forms of nsb_device.cuh (dot3, cross3)
inline float dot3c(V3 a, V3 b) { return fmaf(a.x, b.x, fmaf(a.y, b.y, a.z * b.z)); }
inline V3 cross3c(V3 a, V3 b) { return v3(fmaf(a.y, b.z, -(a.z * b.y)), fmaf(a.z, b.x, -(a.x * b.z)), fmaf(a.x, b.y, -(a.y * b.x))); }
inline V3 normalized3(V3 v) {
	const float n2 = dot3c(v, v);
	if (!(n2 > 0.0f)) return v;
	const float n = sqrtf(n2);
	return v3(v.x / n, v.y / n, v.z / n);
}

}  // namespace

extern "C" {

// coords: n x 7 floats. dfeat_in (may be NULL): fp16 [32 x n] to run the grid backward on instead of the MLP's; grad: n x 3;
// dfeat_out (may be NULL): fp16 [32 x n]; dens_out (may be NULL): fp16 [n].
int orc_density_gradient(const OrcScene* s, const float* coords, uint32_t n, const uint16_t* dfeat_in, float* grad, uint16_t* dfeat_out, uint16_t* dens_out) {
	Model m;
	if (!model_init(m, &s->desc, s->params, s->n_params)) return 1;
#pragma omp parallel for schedule(static)
	for (int64_t i = 0; i < (int64_t)n; ++i) {
		const float* x = coords + 7 * i;
		uint16_t dens, df[32];
		density_backward(m, v3(x[0], x[1], x[2]), &dens, df);
		if (dfeat_in)
			for (int k = 0; k < 32; ++k) df[k] = dfeat_in[(size_t)k * n + i];
		grid_backward(m, x, df, grad + 3 * i);
		if (dfeat_out)
			for (int k = 0; k < 32; ++k) dfeat_out[(size_t)k * n + i] = df[k];
		if (dens_out) dens_out[i] = dens;
	}
	return 0;
}

// float64, no rounding: the raw density at n positions (n x 3, warped) and, when grad is not NULL, its analytic gradient (n x 3)
int orc_density_f64(const OrcScene* s, const double* pos, uint32_t n, double* dens, double* grad) {
	Model m;
	if (!model_init(m, &s->desc, s->params, s->n_params)) return 1;
#pragma omp parallel for schedule(static)
	for (int64_t i = 0; i < (int64_t)n; ++i) dens[i] = density_f64(m, pos + 3 * i, grad ? grad + 3 * i : nullptr);
	return 0;
}

// The opt gradient of Testbed::optimise_mesh_step: compute_mesh_1ring summed per vertex in ascending triangle order, then
// compute_mesh_opt_gradients_kernel with the contractions nvcc makes of it (read off the SASS of the reference's kernel): sg = fma(-1/w, sum, v),
// g = fma(-nn, k_inflate, fma(n*sign, k_density, sg*k_smooth)). k = {thresh, smooth, density, inflate}. dens: fp16 [n_rows], grad: [n_rows x 3].
// Out (any may be NULL): the 1-ring sums [n_rows x 4] (x, y, z, w), normals [n_rows x 3], opt gradient [n_rows x 3].
int orc_mesh_opt_gradient(uint32_t n_rows, const float* pos, const uint32_t* indices, uint32_t n_tris, const uint16_t* dens, const float* grad,
                          const float* k, float* sums_out, float* normals, float* grad_out) {
	std::vector<V3> sum(n_rows, v3(0, 0, 0)), nrm(n_rows, v3(0, 0, 0));
	std::vector<float> wsum(n_rows, 0.0f);
	auto P = [&](uint32_t i) { return v3(pos[3 * i], pos[3 * i + 1], pos[3 * i + 2]); };
	for (uint32_t t = 0; t < n_tris; ++t) {
		const uint32_t ia = indices[3 * t], ib = indices[3 * t + 1], ic = indices[3 * t + 2];
		const V3 pa = P(ia), pb = P(ib), pc = P(ic);
		sum[ia] = add3(sum[ia], add3(pb, pc));
		sum[ib] = add3(sum[ib], add3(pa, pc));
		sum[ic] = add3(sum[ic], add3(pb, pa));
		wsum[ia] += 2.0f; wsum[ib] += 2.0f; wsum[ic] += 2.0f;
		const V3 n = cross3c(sub3(pb, pa), sub3(pa, pc));
		nrm[ia] = add3(nrm[ia], n); nrm[ib] = add3(nrm[ib], n); nrm[ic] = add3(nrm[ic], n);
	}
	for (uint32_t v = 0; v < n_rows; ++v) {
		if (sums_out) { sums_out[4 * v] = sum[v].x; sums_out[4 * v + 1] = sum[v].y; sums_out[4 * v + 2] = sum[v].z; sums_out[4 * v + 3] = wsum[v]; }
		if (normals) { normals[3 * v] = nrm[v].x; normals[3 * v + 1] = nrm[v].y; normals[3 * v + 2] = nrm[v].z; }
		float w = wsum[v];
		if (w <= 0.0f) w = 1.0f;
		const float inv = 1.0f / w;
		const V3 src = P(v);
		const V3 sg = v3(fmaf(-inv, sum[v].x, src.x), fmaf(-inv, sum[v].y, src.y), fmaf(-inv, sum[v].z, src.z));
		const V3 n = normalized3(v3(grad[3 * v], grad[3 * v + 1], grad[3 * v + 2]));
		const V3 nn = normalized3(nrm[v]);
		// the sign of dens - thresh as the device takes it: a NaN difference is the GPU's canonical NaN, whose sign bit is clear, so it counts
		// as +1 whatever the signs of its NaN operands (the host's subtraction would pass a -NaN threshold's sign through)
		const float d = h2f(dens[v]) - k[0];
		const float sgn = std::isnan(d) ? 1.0f : copysignf(1.0f, d);
		if (grad_out) {
			grad_out[3 * v] = fmaf(-nn.x, k[3], fmaf(n.x * sgn, k[2], sg.x * k[1]));
			grad_out[3 * v + 1] = fmaf(-nn.y, k[3], fmaf(n.y * sgn, k[2], sg.y * k[1]));
			grad_out[3 * v + 2] = fmaf(-nn.z, k[3], fmaf(n.z * sgn, k[2], sg.z * k[1]));
		}
	}
	return 0;
}

// tcnn Adam (learning rate 1e-4, beta1 0.9, beta2 0.99, epsilon 1e-8) on n coordinates, each a non-matrix parameter: skipped while its gradient
// is 0, its own step counter. Published adam_step: effective_learning_rate = lr_t / (sqrtf(v) + epsilon), new = weight - effective_learning_rate * m,
// with the moment updates and the subtraction contracted as nvcc does. m1, m2, steps: in/out.
// pows (may be NULL): [n_pows x 2] floats, row t = {powf(0.9f, t), powf(0.99f, t)} as the device computes them (tcnn runs powf on the GPU;
// the host's powf is not correctly rounded and need not agree with it). NULL: the host's powf. Returns 2 when a step count reaches n_pows.
int orc_adam_step(uint32_t n, const float* x_in, const float* g, float* m1, float* m2, uint32_t* steps, float* x_out, const float* pows, uint32_t n_pows) {
	const float B1 = 0.9f, B2 = 0.99f, LR = 1e-4f, EPS = 1e-8f;
	for (uint32_t j = 0; j < n; ++j) {
		float x = x_in[j];
		if (g[j] != 0.0f) {
			m1[j] = fmaf(B1, m1[j], (1.0f - B1) * g[j]);
			m2[j] = fmaf(B2, m2[j], (1.0f - B2) * (g[j] * g[j]));
			const uint32_t t = ++steps[j];
			if (pows && t >= n_pows) return 2;
			const float p1 = pows ? pows[2 * (size_t)t] : powf(B1, (float)t), p2 = pows ? pows[2 * (size_t)t + 1] : powf(B2, (float)t);
			const float lr = LR * (sqrtf(1.0f - p2) / (1.0f - p1));
			const float eff = lr / (sqrtf(m2[j]) + EPS);
			x = fmaf(-eff, m1[j], x);
		}
		x_out[j] = x;
	}
	return 0;
}

// One step of Testbed::optimise_mesh_step after the network: orc_mesh_opt_gradient, then orc_adam_step on every coordinate of the n_rows rows.
int orc_mesh_opt_step(uint32_t n_rows, const float* pos, const uint32_t* indices, uint32_t n_tris, const uint16_t* dens, const float* grad, const float* k,
                      float* m1, float* m2, uint32_t* steps, float* pos_out, float* normals, const float* pows, uint32_t n_pows) {
	std::vector<float> g(3 * (size_t)n_rows);
	orc_mesh_opt_gradient(n_rows, pos, indices, n_tris, dens, grad, k, nullptr, normals, g.data());
	return orc_adam_step(3 * n_rows, pos, g.data(), m1, m2, steps, pos_out, pows, n_pows);
}

}  // extern "C"
