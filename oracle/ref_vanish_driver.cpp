// ref_vanish_driver.cpp — a C entry point around the reference's OWN TetMesh::vanish (tet_mesh.cu:237-363), compiled for the CPU.
//
// TEST INFRASTRUCTURE ONLY: built by oracle/ref_vanish_build.py into oracle/_ref/libnerfshop_ref_vanish.so, loaded by tests/ (and
// nothing else). Reference code here: everything ref_driver.cpp compiles, and tet_mesh_vanish.inc (the clear_cells static, clear_grid
// and TetMesh::vanish, cut out at build time). Ours: ref_driver.cpp and this file's marshalling.
#include "ref_driver.cpp"

#include <chrono>

#include "tet_mesh_vanish.inc"

extern "C" {

// Builds a TetMesh the way ref_tet_mesh_build does (constructor, deformed vertices, post_update_vertices) and runs vanish on the given
// grid (float[5*128^3]) and bitfield (uint8[5*128^3/8]) in place. *seconds: wall time of vanish alone (marking threads, the list, its
// upload and clear_grid).
int ref_tet_mesh_vanish(const float* original_vertices, const float* deformed_vertices, uint32_t n_v, const uint32_t* tets, uint32_t n_tets, const float* amin,
                        const float* amax, float* grid, uint8_t* bitfield, double* seconds) {
	try {
		std::vector<Eigen::Vector3f> ov(n_v);
		for (uint32_t i = 0; i < n_v; ++i) ov[i] = Eigen::Vector3f(original_vertices[3 * i], original_vertices[3 * i + 1], original_vertices[3 * i + 2]);
		std::vector<uint32_t> indices, tt(tets, tets + 4 * (size_t)n_tets);
		TetMesh<float, Eigen::Vector3f> mesh(ov, indices, tt, bb(amin, amax));
		for (uint32_t i = 0; i < n_v; ++i) mesh.vertices[i] = Eigen::Vector3f(deformed_vertices[3 * i], deformed_vertices[3 * i + 1], deformed_vertices[3 * i + 2]);
		mesh.post_update_vertices();
		mesh.original_tet_lut_idx.resize(1);  // the canonical grid plays no part in vanish: skip building it (vanish only checks size() == 0)
		const auto t0 = std::chrono::steady_clock::now();
		mesh.vanish(grid, bitfield, nullptr);
		if (seconds) *seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
		return 0;
	} catch (const std::exception& e) {
		fprintf(stderr, "ref_tet_mesh_vanish: %s\n", e.what());
		return 1;
	}
}

}  // extern "C"
