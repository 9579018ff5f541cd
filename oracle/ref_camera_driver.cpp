// ref_camera_driver.cpp — the reference's OWN camera-path code (camera_path.h: CameraKeyframe, CameraPath; camera_path.cu: lerp, spline),
// cut out by oracle/ref_camera_build.py and compiled for the CPU by g++ with -ffp-contract=off (host code in the reference) into
// oracle/_ref/libnerfshop_ref_camera.so. TEST INFRASTRUCTURE ONLY (tests/test_camera_path_cpu.py pins nerfshop_b200/camera_path.py to it).
// Eigen is the stand-in of oracle/ref_shim_camera/ (the reference's Eigen is absent from its tree).
#include <Eigen/Dense>

#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

namespace tcnn {
template <typename T> T clamp(T v, T lo, T hi) { return v < lo ? lo : (hi < v ? hi : v); }
}
#define NGP_NAMESPACE_BEGIN namespace ngp {
#define NGP_NAMESPACE_END }

NGP_NAMESPACE_BEGIN
#include "camera_path_h.inc"
using namespace Eigen;
#include "camera_path_cu.inc"
NGP_NAMESPACE_END

using namespace ngp;

static CameraKeyframe kf(const float* v) {  // R[4], T[3], slice, scale, fov, dof
	return CameraKeyframe(Eigen::Vector4f(v[0], v[1], v[2], v[3]), Eigen::Vector3f(v[4], v[5], v[6]), v[7], v[8], v[9], v[10]);
}
static void put(const CameraKeyframe& k, float* out) {
	for (int i = 0; i < 4; ++i) out[i] = k.R[i];
	for (int i = 0; i < 3; ++i) out[4 + i] = k.T[i];
	out[7] = k.slice; out[8] = k.scale; out[9] = k.fov; out[10] = k.dof;
}

extern "C" {
// CameraKeyframe::m(): 12 floats column-major
void refcam_m(const float* v, float* out) {
	const Eigen::Matrix<float, 3, 4> m = kf(v).m();
	for (int i = 0; i < 12; ++i) out[i] = m.a[i];
}
// CameraKeyframe(Matrix<float, 3, 4>, sl, sc, fv, df): m column-major -> 11 floats
void refcam_from_matrix(const float* m, float sl, float sc, float fv, float df, float* out) {
	Eigen::Matrix<float, 3, 4> mm;
	for (int i = 0; i < 12; ++i) mm.a[i] = m[i];
	put(CameraKeyframe(mm, sl, sc, fv, df), out);
}
// CameraPath::eval_camera_path(t) over n keyframes (11 floats each) at n_t times -> 11 floats per time
void refcam_eval(const float* kfs, int n, const float* ts, int n_t, float* out) {
	CameraPath p;
	for (int i = 0; i < n; ++i) p.m_keyframes.push_back(kf(kfs + 11 * i));
	for (int i = 0; i < n_t; ++i) put(p.eval_camera_path(ts[i]), out + 11 * i);
}
}
