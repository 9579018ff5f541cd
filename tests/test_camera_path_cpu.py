"""Camera paths on the host (nerfshop_b200/camera_path.py): keyframe arithmetic, the B-spline path, the JSON file, the log_space_lerp
restatement against a float64 matrix logarithm / exponential, and render_to_cpu's sub-frame sequence against a literal transcription of
python_api.cu:129-175. No GPU."""
import json
import os

import numpy as np
import pytest
import scipy.linalg
from scipy.spatial.transform import Rotation

from nerfshop_b200 import abi
from nerfshop_b200 import camera_path as cp

f32 = np.float32


def _rigid(rng, angle=None):
    if angle is None:
        R = Rotation.random(random_state=rng).as_matrix()
    else:
        axis = rng.standard_normal(3)
        R = Rotation.from_rotvec(axis / np.linalg.norm(axis) * angle).as_matrix()
    m = np.zeros((3, 4))
    m[:, :3] = R
    m[:, 3] = rng.uniform(-2, 2, 3)
    return m.astype(f32)


def _h(m):
    out = np.eye(4)
    out[:3, :] = m
    return out


def _rigidity(m):
    R = m[:, :3].astype(np.float64)
    return max(np.abs(R.T @ R - np.eye(3)).max(), abs(np.linalg.det(R) - 1.0))


# ---- keyframes ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("branch", ["trace", "x", "y", "z"])
def test_matrix_to_keyframe_and_back(branch):
    """Every branch of Eigen's quaternion-from-matrix (trace > 0, else the largest diagonal) gives a unit quaternion whose m() is the
    matrix to float32 precision."""
    rng = np.random.default_rng(7)
    n = 0
    while n < 50:
        m = _rigid(rng)
        d = np.diag(m[:, :3])
        tr = f32(f32(d[0] + d[1]) + d[2])
        got = "trace" if tr > 0 else "xyz"[int(np.argmax(d))]
        if got != branch:
            continue
        n += 1
        k = cp.CameraKeyframe.from_matrix(m, 0.1, 1.2, 40.0, 0.01)
        assert abs(np.linalg.norm(k.R.astype(np.float64)) - 1) < 1e-6
        assert np.abs(k.m() - m).max() < 1e-6
        assert k.m().dtype == np.float32 and np.array_equal(k.m()[:, 3], m[:, 3])
        assert (k.slice, k.scale, k.fov, k.dof) == (f32(0.1), f32(1.2), f32(40.0), f32(0.01))


def test_m_normalises_and_follows_eigen():
    rng = np.random.default_rng(8)
    for _ in range(50):
        q = rng.standard_normal(4).astype(f32) * f32(rng.uniform(0.1, 10))
        k = cp.CameraKeyframe(q, rng.standard_normal(3))
        R = Rotation.from_quat(q.astype(np.float64)).as_matrix()  # scipy: (x, y, z, w), normalised
        assert np.abs(k.m()[:, :3] - R).max() < 1e-6
        assert _rigidity(k.m()) < 1e-6
    # the same quaternion in the other hemisphere is the same rotation
    assert np.array_equal(cp.CameraKeyframe(-q).m(), cp.CameraKeyframe(q).m())


def test_plus_takes_the_short_path_and_times_scales():
    a = cp.CameraKeyframe([0, 0, 0, 1], [1, 2, 3], 0.5, 1.0, 50.0, 0.1)
    b = cp.CameraKeyframe([0, 0, 0, -1], [1, 1, 1], 0.25, 2.0, 40.0, 0.0)
    s = a + b
    assert np.array_equal(s.R, np.array([0, 0, 0, 2], f32)) and np.array_equal(s.T, np.array([2, 3, 4], f32))
    assert (s.slice, s.scale, s.fov, s.dof) == (f32(0.75), f32(3.0), f32(90.0), f32(0.1))
    h = a * 0.5
    assert np.array_equal(h.R, np.array([0, 0, 0, 0.5], f32)) and h.fov == f32(25.0)


@pytest.mark.parametrize("n", [2, 3, 4, 7])
def test_eval_camera_path(n):
    """t *= n - 1, clamped neighbours and the B-spline weights: at a keyframe time the path is (p[i-1] + 4 p[i] + p[i+1]) / 6 of the
    clamped neighbours; the weights sum to one; identical keyframes give that keyframe back (to rounding)."""
    rng = np.random.default_rng(n)
    kfs = []
    for i in range(n):
        q = Rotation.random(random_state=rng).as_quat().astype(f32)
        if i % 2:
            q = -q  # both hemispheres
        kfs.append(cp.CameraKeyframe(q, rng.uniform(-1, 1, 3), rng.uniform(0, 1), rng.uniform(0.5, 2), rng.uniform(30, 70), rng.uniform(0, 0.1)))
    path = cp.CameraPath(kfs)
    for i in range(n):
        t = i / (n - 1)
        got = path.eval_camera_path(t)
        p0, p1, p2 = path.get_keyframe(i - 1), path.get_keyframe(i), path.get_keyframe(i + 1)
        for name in ("slice", "scale", "fov", "dof"):
            want = (getattr(p0, name) + 4 * getattr(p1, name) + getattr(p2, name)) / 6
            assert abs(float(getattr(got, name)) - float(want)) < 1e-5 * max(1.0, abs(float(want)))
        assert np.abs(got.T - (p0.T + 4 * p1.T + p2.T) / 6).max() < 1e-5
    for t in np.concatenate([[0.0, 1.0], rng.uniform(0, 1, 20)]):
        k = path.eval_camera_path(t)
        assert k.R.dtype == np.float32 and np.isfinite(k.R).all() and _rigidity(k.m()) < 1e-6
    same = cp.CameraPath([kfs[0]] * 4)
    k = same.eval_camera_path(0.37)
    assert np.abs(k.m() - kfs[0].m()).max() < 1e-6 and abs(k.fov - kfs[0].fov) < 1e-4


def test_save_and_load_round_trip(tmp_path):
    rng = np.random.default_rng(3)
    kfs = [cp.CameraKeyframe(Rotation.random(random_state=rng).as_quat(), rng.uniform(-1, 1, 3), 0.1 * i, 1.0, 50.625, 0.0) for i in range(3)]
    path = cp.CameraPath(kfs, playtime=0.3)
    fn = str(tmp_path / "path.json")
    path.save(fn)
    j = json.load(open(fn))
    assert set(j) == {"time", "path"} and set(j["path"][0]) == {"R", "T", "slice", "scale", "fov", "dof"} and len(j["path"][0]["R"]) == 4
    back = cp.CameraPath.load(fn)
    assert back.playtime == f32(0.3)
    for a, b in zip(kfs, back.keyframes):
        assert np.array_equal(a.R, b.R) and np.array_equal(a.T, b.T) and (a.slice, a.scale, a.fov, a.dof) == (b.slice, b.scale, b.fov, b.dof)
    (tmp_path / "bare.json").write_text(json.dumps({"path": j["path"][:1]}))  # "time" is optional
    assert len(cp.CameraPath.load(str(tmp_path / "bare.json")).keyframes) == 1
    with pytest.raises(FileNotFoundError):
        cp.CameraPath.load(str(tmp_path / "missing.json"))


def test_focal_length_from_fov():
    """set_fov + calc_focal_length: m_relative_focal_length = 0.5 / tanf(0.5 * fov * PI / 180), times resolution[fov_axis] * zoom."""
    st = cp.CameraState()
    st.set_camera_from_keyframe(cp.CameraKeyframe(fov=90.0, slice=0.25, scale=1.5, dof=0.02))
    fl = st.focal_length(1920, 1080)
    assert abs(float(fl[0]) - 540.0) < 1e-3 and fl[0] == fl[1]
    st.fov_axis, st.zoom = 0, 2.0
    assert abs(float(st.focal_length(1920, 1080)[0]) - 1920.0) < 1e-2
    f = cp.frame_from_keyframe(abi.NsbFrame(width=320, height=180), cp.CameraKeyframe(fov=90.0, slice=0.25, scale=1.5, dof=0.02))
    assert f.focus_z == 1.75 and f.dof == pytest.approx(0.02) and f.focal_length[1] == pytest.approx(90.0, abs=1e-4)
    assert list(f.camera0) == list(f.camera1)


# ---- log_space_lerp ---------------------------------------------------------------------------------------------------------------------
def _pairs(rng, n=40, near_pi=True):
    out = [(_rigid(rng), _rigid(rng)) for _ in range(n)]
    # relative rotations near pi and near 0. Closer to pi than ~1e-3 the matrix logarithm of the float32-rounded pair is ill-conditioned
    # (its sensitivity grows as 1 / sin(angle) while the rounded rotations are orthonormal to ~1e-7), and float64 logm and the
    # closed form then part by more than 1e-5: one such pair is kept for the rigidity and endpoint checks only (near_pi=False skips it)
    for angle in (np.pi - 5e-2, np.pi - 1e-2, np.pi - 3e-3, 1e-4, 1e-7, 0.0) + ((np.pi - 1e-4,) if near_pi else ()):
        A = _rigid(rng)
        D = _rigid(rng, angle)
        out.append((A, (_h(D) @ _h(A))[:3].astype(f32)))
    return out


def test_log_space_lerp_endpoints_and_rigidity():
    rng = np.random.default_rng(11)
    for A, B in _pairs(rng):
        assert np.array_equal(cp.log_space_lerp(A, B, 0.0), A)
        assert np.abs(cp.log_space_lerp(A, B, 1.0) - B).max() <= 2e-6
        for t in (0.25, 0.5, 0.9):
            assert _rigidity(cp.log_space_lerp(A, B, t)) <= 1e-6


def test_log_space_lerp_matches_matrix_log_and_exp():
    """((B A^-1).log() * t).exp() * A with scipy's float64 logm / expm."""
    rng = np.random.default_rng(12)
    worst = 0.0
    for A, B in _pairs(rng, near_pi=False):
        L = scipy.linalg.logm(_h(B) @ np.linalg.inv(_h(A)))
        assert np.abs(L.imag).max() < 1e-9 if np.iscomplexobj(L) else True
        L = np.real(L)
        for t in (0.1, 0.5, 0.77):
            want = (scipy.linalg.expm(L * t) @ _h(A))[:3]
            worst = max(worst, np.abs(cp.log_space_lerp(A, B, t) - want).max())
    print(f"log_space_lerp vs logm/expm: L-inf {worst:.2e}")
    assert worst <= 1e-5


def test_camera_smoothing():
    rng = np.random.default_rng(13)
    st = cp.CameraState(camera=_rigid(rng), smoothed_camera=_rigid(rng))
    cp.apply_camera_smoothing(st, 1000.0 / 30)
    assert np.array_equal(st.smoothed_camera, st.camera)  # smoothing off: the camera itself
    st = cp.CameraState(camera=_rigid(rng), smoothed_camera=_rigid(rng), camera_smoothing=True)
    prev = st.smoothed_camera.copy()
    cp.apply_camera_smoothing(st, 1000.0 / 30)
    decay = f32(0.02) ** (f32(1000.0 / 30) / f32(1000))
    assert np.abs(st.smoothed_camera - cp.log_space_lerp(prev, st.camera, f32(1) - decay)).max() == 0


# ---- render_to_cpu's sub-frames ---------------------------------------------------------------------------------------------------------
class _Testbed:
    """python_api.cu:129-175 transcribed line by line over the module's primitives (the cameras, times and spp indices it renders)."""

    def __init__(self, path, state):
        self.m_camera_path, self.s = path, state
        self.rendered = []

    def set_camera_from_time(self, t):
        if not self.m_camera_path.keyframes:
            return
        self.s.set_camera_from_keyframe(self.m_camera_path.eval_camera_path(t))

    def render_to_cpu(self, width, height, spp, linear, start_time, end_time, fps, shutter_fraction):
        start_time, end_time, fps, shutter_fraction = f32(start_time), f32(end_time), f32(fps), f32(shutter_fraction)
        if end_time < f32(0):
            end_time = start_time
        start_cam_matrix = self.s.smoothed_camera.copy()
        if start_time >= f32(0):
            self.set_camera_from_time(end_time)
            cp.apply_camera_smoothing(self.s, f32(1000) / fps)
        else:
            start_cam_matrix = self.s.smoothed_camera = self.s.camera.copy()
        end_cam_matrix = self.s.smoothed_camera.copy()
        for i in range(spp):
            start_alpha = f32(i) / f32(spp) * shutter_fraction
            end_alpha = (f32(i) + f32(1)) / f32(spp) * shutter_fraction
            sample_start = cp.log_space_lerp(start_cam_matrix, end_cam_matrix, start_alpha)
            sample_end = cp.log_space_lerp(start_cam_matrix, end_cam_matrix, end_alpha)
            if start_time >= f32(0):
                self.set_camera_from_time(start_time + (end_time - start_time) * (start_alpha + end_alpha) / f32(2))
                self.s.smoothed_camera = self.s.camera.copy()
            fl = self.s.focal_length(width, height)
            self.rendered.append((sample_start, sample_end, i, fl, f32(self.s.slice_plane_z) + f32(self.s.scale), f32(self.s.dof)))
        self.s.smoothed_camera = end_cam_matrix


def _cam(vals):
    return np.array(vals, f32).reshape(4, 3).T


@pytest.mark.parametrize("smoothing", [False, True])
@pytest.mark.parametrize("times", [(0.0, 0.1), (0.35, 0.5), (0.9, -1.0), (-1.0, -1.0)])
def test_sub_frames_follow_render_to_cpu(smoothing, times):
    rng = np.random.default_rng(5)
    path = cp.CameraPath([cp.CameraKeyframe.from_matrix(_rigid(rng), rng.uniform(0, 0.3), rng.uniform(0.8, 1.2), rng.uniform(40, 60), rng.uniform(0, 0.05))
                          for _ in range(4)])
    start = _rigid(rng)
    st_a = cp.CameraState(camera=start.copy(), smoothed_camera=start.copy(), camera_smoothing=smoothing)
    st_b = cp.CameraState(camera=start.copy(), smoothed_camera=start.copy(), camera_smoothing=smoothing)
    tb = _Testbed(path, st_b)
    base = abi.NsbFrame(width=320, height=180)
    for frame_no in range(3):  # consecutive frames carry m_smoothed_camera
        t0 = times[0] + 0.1 * frame_no if times[0] >= 0 else times[0]
        t1 = times[1] + 0.1 * frame_no if times[1] >= 0 else times[1]
        frames, end_cam = cp.sub_frames(path, t0, t1, 30.0, 5, 0.5, st_a, base)
        tb.rendered = []
        tb.render_to_cpu(320, 180, 5, True, t0, t1, 30.0, 0.5)
        assert len(frames) == 5
        for f, (c0, c1, i, fl, focus, dof) in zip(frames, tb.rendered):
            assert np.array_equal(_cam(f.camera0), c0) and np.array_equal(_cam(f.camera1), c1)
            assert f.spp_index == i and list(f.rolling_shutter) == [0.0] * 4
            assert f32(f.focal_length[0]) == fl[0] and f32(f.focal_length[1]) == fl[1] and f32(f.focus_z) == focus and f32(f.dof) == dof
        assert np.array_equal(end_cam, st_b.smoothed_camera) and np.array_equal(st_a.smoothed_camera, st_b.smoothed_camera)
        assert np.array_equal(st_a.camera, st_b.camera)


def test_cpp_shim_keyframes_match_the_python_module(built_lib, tmp_path):
    """ngp_b200::CameraKeyframe / CameraPath (nerfshop_host.hpp, g++ without FMA contraction) and camera_path.py compute the same floats,
    bit for bit: m(), the matrix constructor on every branch and eval_camera_path on 2-7 keyframes in both quaternion hemispheres."""
    import os
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "kf.cpp"
    src.write_text(
        '#include "nerfshop_b200/host/nerfshop_host.hpp"\n#include <cstdio>\n'
        "int main() {\n  int n; std::scanf(\"%d\", &n); ngp_b200::CameraPath p;\n"
        "  for (int i = 0; i < n; ++i) { ngp_b200::CameraKeyframe k; float v[11]; for (float& x : v) std::scanf(\"%a\", &x);\n"
        "    for (int c = 0; c < 4; ++c) k.R[c] = v[c]; for (int c = 0; c < 3; ++c) k.T[c] = v[4 + c]; k.slice = v[7]; k.scale = v[8]; k.fov = v[9]; k.dof = v[10];\n"
        "    p.m_keyframes.push_back(k); float m[12]; k.m(m); for (float x : m) std::printf(\"%a \", x);\n"
        "    auto b = ngp_b200::CameraKeyframe::from_matrix(m, 0.f, 1.f, 50.f, 0.f); for (float x : b.R) std::printf(\"%a \", x); std::printf(\"\\n\"); }\n"
        "  int nt; std::scanf(\"%d\", &nt);\n"
        "  for (int i = 0; i < nt; ++i) { float t; std::scanf(\"%a\", &t); auto k = p.eval_camera_path(t);\n"
        "    for (float x : k.R) std::printf(\"%a \", x); for (float x : k.T) std::printf(\"%a \", x);\n"
        "    std::printf(\"%a %a %a %a\\n\", k.slice, k.scale, k.fov, k.dof); }\n  return 0;\n}\n")
    exe = tmp_path / "kf"
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-std=c++17", "-O2", "-ffp-contract=off", "-I", root, str(src), "-o", str(exe)], check=True)
    rng = np.random.default_rng(21)
    for n in (2, 3, 4, 7):
        kfs = []
        for i in range(n):
            q = (Rotation.random(random_state=rng).as_quat() * rng.uniform(0.5, 2)).astype(f32)
            kfs.append(cp.CameraKeyframe(-q if i % 2 else q, rng.uniform(-1, 1, 3), rng.uniform(0, 1), rng.uniform(0.5, 2), rng.uniform(30, 70), rng.uniform(0, 0.1)))
        ts = np.concatenate([[0.0, 1.0], np.arange(n) / max(n - 1, 1), rng.uniform(0, 1, 10)]).astype(f32)
        lines = [str(n)] + [" ".join(float(v).hex() for v in np.concatenate([k.R, k.T, [k.slice, k.scale, k.fov, k.dof]]).astype(f32)) for k in kfs]
        lines += [str(ts.size), " ".join(float(t).hex() for t in ts)]
        out = subprocess.run([str(exe)], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout.split("\n")
        path = cp.CameraPath(kfs)
        for i, k in enumerate(kfs):
            got = np.array([float.fromhex(v) for v in out[i].split()], f32)
            m = k.m()
            assert np.array_equal(got[:12], m.T.reshape(-1)), (n, i)
            assert np.array_equal(got[12:], cp.CameraKeyframe.from_matrix(m).R), (n, i)
        for j, t in enumerate(ts):
            got = np.array([float.fromhex(v) for v in out[n + j].split()], f32)
            k = path.eval_camera_path(t)
            assert np.array_equal(got, np.concatenate([k.R, k.T, [k.slice, k.scale, k.fov, k.dof]]).astype(f32)), (n, float(t))


# ---- against the reference's own camera_path.h / camera_path.cu (oracle/_ref/libnerfshop_ref_camera.so, replayed where absent) --------
def _ref_camera_available():
    from oracle import ref_camera_build

    return ref_camera_build.build() is not None


def _rows(kfs):
    return np.array([np.concatenate([k.R, k.T, [k.slice, k.scale, k.fov, k.dof]]) for k in kfs], f32)


@pytest.mark.skipif(not (_ref_camera_available() or os.path.isdir(os.path.join(os.path.dirname(__file__), "golden", "ref", "test_camera_path_cpu"))),
                    reason="neither oracle/_ref nor stored reference results (tests/golden/ref/)")
@pytest.mark.parametrize("n", [2, 3, 4, 7])
def test_keyframes_bit_identical_to_reference(n):
    """m(), the matrix constructor (all four branches of the quaternion-from-matrix) and eval_camera_path at t = 0, 1, the keyframe
    times and random times, on keyframes in both quaternion hemispheres and of any norm: the reference's compiled code, bit for bit."""
    import ref_golden

    from oracle import ref_camera

    have = _ref_camera_available()
    rng = np.random.default_rng(100 + n)
    kfs = []
    for i in range(n):
        q = (Rotation.random(random_state=rng).as_quat() * rng.uniform(0.5, 2.0)).astype(f32)
        kfs.append(cp.CameraKeyframe(-q if i % 2 else q, rng.uniform(-1, 1, 3), rng.uniform(0, 1), rng.uniform(0.5, 2), rng.uniform(30, 70), rng.uniform(0, 0.1)))
    rows = _rows(kfs)
    ts = np.concatenate([[0.0, 1.0], np.arange(n) / (n - 1), rng.uniform(0, 1, 24)]).astype(f32)
    # matrices for every branch: trace > 0, and the largest diagonal entry at x, y and z
    mats, seen = [], set()
    while len(mats) < 64:
        m = _rigid(rng)
        d = np.diag(m[:, :3])
        b = "trace" if f32(f32(d[0] + d[1]) + d[2]) > 0 else "xyz"[int(np.argmax(d))]
        if sum(1 for x in seen if x[0] == b) < 16:
            seen.add((b, len(mats)))
            mats.append(m.T.reshape(-1))
    mats = np.array(mats, f32)
    assert {x[0] for x in seen} == {"trace", "x", "y", "z"}

    want_m = ref_golden._call(have, ref_camera.m, rows)
    want_k = ref_golden._call(have, ref_camera.from_matrix, mats)
    want_e = ref_golden._call(have, ref_camera.eval_camera_path, rows, ts)
    got_m = np.array([k.m().T.reshape(-1) for k in kfs], f32)
    got_k = _rows([cp.CameraKeyframe.from_matrix(mm.reshape(4, 3).T, 0.0, 1.0, 50.0, 0.0) for mm in mats])
    path = cp.CameraPath(kfs)
    got_e = _rows([path.eval_camera_path(t) for t in ts])
    for name, g, w in (("m()", got_m, want_m), ("matrix -> keyframe", got_k, want_k), ("eval_camera_path", got_e, want_e)):
        assert np.array_equal(g.view(np.uint32), np.asarray(w, f32).view(np.uint32)), name


def test_cpp_shim_render_to_cpu_compiles_with_the_cuda_runtime(tmp_path):
    """ngp_b200::render_to_cpu is compiled only where cuda_runtime_api.h is on the include path: compile a caller against it."""
    import subprocess

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    inc = "/usr/local/cuda/include"
    if not os.path.exists(os.path.join(inc, "cuda_runtime_api.h")):
        pytest.skip("no CUDA runtime headers")
    src = tmp_path / "r2c.cpp"
    src.write_text('#include "nerfshop_b200/host/nerfshop_host.hpp"\n'
                   "#ifndef NSB_HOST_HAVE_CUDART\n#error the CUDA runtime header was not found\n#endif\n"
                   "void f(ngp_b200::Context& c, const std::vector<NsbFrame>& fr, const NsbTonemap& tm, float* a, float* o, float* h) {\n"
                   "  ngp_b200::render_to_cpu(c, fr, tm, a, o, h, nullptr);\n}\n")
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-std=c++17", "-c", "-I", root, "-I", inc, str(src), "-o", str(tmp_path / "r2c.o")], check=True)
