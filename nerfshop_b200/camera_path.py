"""Camera paths and videos: the reference's keyframe paths, render_to_cpu's sub-frames with shutter, and run.py's video frames.

  CameraKeyframe                <- CameraKeyframe (camera_path.h:30-62): m(), the matrix constructor, + and *
  spline / CameraPath           <- spline (camera_path.cu:52-70, the cubic B-spline branch it compiles), CameraPath::eval_camera_path
                                   (camera_path.h:71-78), CameraPath::save / load (camera_path.cu:108-145) with their JSON
  frame_from_keyframe           <- Testbed::set_camera_from_keyframe (testbed.cu:2099-2105) + what render_frame hands render_nerf:
                                   set_fov (:2125-2127), fov_to_focal_length (common_device.cuh:444-446), calc_focal_length (:2556-2558),
                                   focus_z = m_slice_plane_z + m_scale, m_dof
  log_space_lerp                <- log_space_lerp (common_device.cu:27-36): a restatement, see its docstring
  apply_camera_smoothing        <- Testbed::apply_camera_smoothing (testbed.cu:2086-2093)
  sub_frames / render           <- Testbed::render_to_cpu (python_api.cu:129-175)
  render_video                  <- scripts/run.py's --video_camera_path loop (run.py:340-356) up to its JPEG files: PNG files here

The keyframe arithmetic is float32 in the reference's operation order, with Eigen's (SSE) reductions: a 4-vector's dot product and squared
norm sum as (x0 + x2) + (x1 + x3); a trace as (m00 + m11) + m22. tanf and powf are the host C library's, called through ctypes, as the
reference's host code calls them. load_relative_to_first is false in the reference and the only case supported here.
"""
from __future__ import annotations

import ctypes as C
import ctypes.util
import json
import math
import os
from dataclasses import dataclass, field

import numpy as np

from . import abi, slices

f32 = np.float32
_libm = C.CDLL(ctypes.util.find_library("m") or "libm.so.6")
_libm.tanf.restype, _libm.tanf.argtypes = C.c_float, [C.c_float]
_libm.powf.restype, _libm.powf.argtypes = C.c_float, [C.c_float, C.c_float]
PI = f32(3.14159265358979323846)  # tcnn::PI() as float


def _dot4(a, b) -> np.float32:
    p = a * b  # float32 products
    return f32(f32(p[0] + p[2]) + f32(p[1] + p[3]))


def _rot_to_quat(m) -> np.ndarray:
    """Eigen's Quaternionf(Matrix3f) (Quaternion.h, quaternionbase_assign_impl<Other, 3, 3>): coeffs (x, y, z, w), float32."""
    m = np.asarray(m, f32)
    q = np.zeros(4, f32)  # x, y, z, w
    t = f32(f32(m[0, 0] + m[1, 1]) + m[2, 2])
    with np.errstate(all="ignore"):
        if t > 0:
            t = np.sqrt(f32(t + f32(1)))
            q[3] = f32(0.5) * t
            t = f32(0.5) / t
            q[0] = f32(m[2, 1] - m[1, 2]) * t
            q[1] = f32(m[0, 2] - m[2, 0]) * t
            q[2] = f32(m[1, 0] - m[0, 1]) * t
        else:
            i = 0
            if m[1, 1] > m[0, 0]:
                i = 1
            if m[2, 2] > m[i, i]:
                i = 2
            j, k = (i + 1) % 3, (i + 2) % 3
            t = np.sqrt(f32(f32(f32(m[i, i] - m[j, j]) - m[k, k]) + f32(1)))
            q[i] = f32(0.5) * t
            t = f32(0.5) / t
            q[3] = f32(m[k, j] - m[j, k]) * t
            q[j] = f32(m[j, i] + m[i, j]) * t
            q[k] = f32(m[k, i] + m[i, k]) * t
    return q


def _quat_to_rot(r) -> np.ndarray:
    """Eigen's Quaternionf(R).normalized().toRotationMatrix(), float32."""
    r = np.asarray(r, f32)
    with np.errstate(all="ignore"):
        n2 = _dot4(r, r)
        x, y, z, w = (r / np.sqrt(n2)) if n2 > 0 else r
        tx, ty, tz = f32(2) * x, f32(2) * y, f32(2) * z
        twx, twy, twz = tx * w, ty * w, tz * w
        txx, txy, txz = tx * x, ty * x, tz * x
        tyy, tyz, tzz = ty * y, tz * y, tz * z
        one = f32(1)
        return np.array([[one - f32(tyy + tzz), txy - twz, txz + twy],
                         [txy + twz, one - f32(txx + tzz), tyz - twx],
                         [txz - twy, tyz + twx, one - f32(txx + tyy)]], f32)


@dataclass
class CameraKeyframe:
    """R: quaternion (x, y, z, w), T: position, slice: m_slice_plane_z, scale: m_scale, fov: degrees along the fov axis, dof: aperture."""
    R: np.ndarray = field(default_factory=lambda: np.array([0, 0, 0, 1], f32))
    T: np.ndarray = field(default_factory=lambda: np.zeros(3, f32))
    slice: np.float32 = f32(0)
    scale: np.float32 = f32(1)
    fov: np.float32 = f32(50.625)
    dof: np.float32 = f32(0)

    def __post_init__(self):
        self.R = np.asarray(self.R, f32).reshape(4).copy()
        self.T = np.asarray(self.T, f32).reshape(3).copy()
        self.slice, self.scale, self.fov, self.dof = f32(self.slice), f32(self.scale), f32(self.fov), f32(self.dof)

    @classmethod
    def from_matrix(cls, m, slice=0.0, scale=1.0, fov=50.625, dof=0.0) -> "CameraKeyframe":
        """CameraKeyframe(Matrix<float, 3, 4>, sl, sc, fv, df): T = column 3, R = Quaternionf(rotation block).coeffs()."""
        m = np.asarray(m, f32).reshape(3, 4)
        return cls(_rot_to_quat(m[:, :3]), m[:, 3], slice, scale, fov, dof)

    def m(self) -> np.ndarray:
        """3x4 camera matrix (row-major numpy; NsbFrame stores it column-major)."""
        out = np.zeros((3, 4), f32)
        out[:, :3] = _quat_to_rot(self.R)
        out[:, 3] = self.T
        return out

    def __mul__(self, f) -> "CameraKeyframe":
        f = f32(f)
        return CameraKeyframe(self.R * f, self.T * f, self.slice * f, self.scale * f, self.fov * f, self.dof * f)

    def __add__(self, rhs: "CameraKeyframe") -> "CameraKeyframe":
        rr = rhs.R
        if _dot4(rr, self.R) < 0:
            rr = -rr
        return CameraKeyframe(self.R + rr, self.T + rhs.T, self.slice + rhs.slice, self.scale + rhs.scale, self.fov + rhs.fov, self.dof + rhs.dof)

    def to_json(self) -> dict:
        return {"R": [float(v) for v in self.R], "T": [float(v) for v in self.T], "slice": float(self.slice), "scale": float(self.scale),
                "fov": float(self.fov), "dof": float(self.dof)}

    @classmethod
    def from_json(cls, j: dict) -> "CameraKeyframe":
        return cls(np.array(j["R"][:4], np.float64).astype(f32), np.array(j["T"][:3], np.float64).astype(f32),
                   j["slice"], j["scale"], j["fov"], j["dof"])


def spline(t, p0: CameraKeyframe, p1: CameraKeyframe, p2: CameraKeyframe, p3: CameraKeyframe) -> CameraKeyframe:
    """The cubic B-spline branch of spline() (camera_path.cu:61-69); the Catmull-Rom branch is compiled out (`if (0)`)."""
    t = f32(t)
    one, sixth = f32(1), f32(1) / f32(6)
    tt = t * t
    ttt = tt * t
    u = one - t
    a = u * u * u * sixth
    b = f32(f32(f32(3) * ttt - f32(6) * tt) + f32(4)) * sixth
    c = f32(f32(f32(f32(-3) * ttt + f32(3) * tt) + f32(3) * t) + one) * sixth
    d = ttt * sixth
    return p0 * a + p1 * b + p2 * c + p3 * d


class CameraPath:
    """CameraPath (camera_path.h:64-97): keyframes, play time, evaluation and the JSON file."""

    def __init__(self, keyframes=None, playtime: float = 0.0):
        self.keyframes = list(keyframes or [])
        self.playtime = f32(playtime)

    def get_keyframe(self, i: int) -> CameraKeyframe:
        return self.keyframes[min(max(i, 0), len(self.keyframes) - 1)]

    def eval_camera_path(self, t) -> CameraKeyframe:
        if not self.keyframes:
            raise ValueError("eval_camera_path: the path has no keyframes")
        t = f32(t) * f32(len(self.keyframes) - 1)
        fl = f32(math.floor(t))
        t1 = int(fl)
        return spline(t - fl, self.get_keyframe(t1 - 1), self.get_keyframe(t1), self.get_keyframe(t1 + 1), self.get_keyframe(t1 + 2))

    def save(self, filename: str) -> None:
        with open(filename, "w") as fh:
            json.dump({"time": float(self.playtime), "path": [k.to_json() for k in self.keyframes]}, fh)

    @classmethod
    def load(cls, filename: str) -> "CameraPath":
        """CameraPath::load with load_relative_to_first = false (the reference's value): keyframes as stored; "time" and "path" optional."""
        if not os.path.exists(filename):
            raise FileNotFoundError(f'Camera path "{filename}" does not exist.')
        with open(filename) as fh:
            j = json.load(fh)
        return cls([CameraKeyframe.from_json(el) for el in j.get("path", [])], j.get("time", 0.0))


# ---- the Testbed members a render reads ------------------------------------------------------------------------------------
def fov_to_focal_length(resolution: int, degrees) -> np.float32:
    """fov_to_focal_length(int, float) (common_device.cuh:444-446): 0.5 * res / tanf(0.5 * degrees * PI / 180) in float32."""
    arg = f32(f32(f32(0.5) * f32(degrees)) * PI) / f32(180)
    return f32(f32(0.5) * f32(resolution)) / f32(_libm.tanf(float(arg)))


@dataclass
class CameraState:
    """The Testbed members render_to_cpu reads and writes: m_camera, m_smoothed_camera, m_camera_smoothing, m_relative_focal_length,
    m_fov_axis, m_zoom, m_slice_plane_z, m_scale, m_dof (defaults testbed.h:462-474, 772)."""
    camera: np.ndarray = field(default_factory=lambda: np.zeros((3, 4), f32))
    smoothed_camera: np.ndarray = field(default_factory=lambda: np.zeros((3, 4), f32))
    camera_smoothing: bool = False
    relative_focal_length: np.ndarray = field(default_factory=lambda: np.ones(2, f32))
    fov_axis: int = 1
    zoom: float = 1.0
    slice_plane_z: float = 0.0
    scale: float = 1.0
    dof: float = 0.0

    def set_camera_from_keyframe(self, k: CameraKeyframe) -> None:
        """Testbed::set_camera_from_keyframe (testbed.cu:2099-2105), set_fov (:2125-2127) included."""
        self.camera = k.m()
        self.slice_plane_z, self.scale, self.dof = f32(k.slice), f32(k.scale), f32(k.dof)
        self.relative_focal_length = np.full(2, fov_to_focal_length(1, k.fov), f32)

    def focal_length(self, width: int, height: int) -> np.ndarray:
        """calc_focal_length (testbed.cu:2556-2558): m_relative_focal_length * resolution[m_fov_axis] * m_zoom."""
        res = (width, height)[self.fov_axis]
        return (self.relative_focal_length * f32(res)) * f32(self.zoom)


def _set_camera(vals, m) -> None:
    flat = np.asarray(m, f32).reshape(3, 4).T.reshape(-1)  # column-major
    for i in range(12):
        vals[i] = float(flat[i])


def frame_from_keyframe(frame: abi.NsbFrame, kf: CameraKeyframe, fov_axis: int = 1, zoom: float = 1.0) -> abi.NsbFrame:
    """A copy of `frame` seen through keyframe kf, as set_camera_from_keyframe then render_frame -> render_nerf pass it: camera0 = camera1 =
    kf.m(), focal length from kf.fov (set_fov, calc_focal_length with fov_axis and zoom: m_fov_axis, m_zoom), focus_z = slice + scale, dof."""
    st = CameraState(fov_axis=fov_axis, zoom=zoom)
    st.set_camera_from_keyframe(kf)
    return _frame_from_state(frame, st, st.camera, st.camera)


def _frame_from_state(frame: abi.NsbFrame, st: CameraState, cam0, cam1) -> abi.NsbFrame:
    f = abi.NsbFrame.from_buffer_copy(frame)
    _set_camera(f.camera0, cam0)
    _set_camera(f.camera1, cam1)
    fl = st.focal_length(f.width, f.height)
    f.focal_length[0], f.focal_length[1] = float(fl[0]), float(fl[1])
    f.focus_z = float(f32(st.slice_plane_z) + f32(st.scale))
    f.dof = float(f32(st.dof))
    return f


# ---- log_space_lerp and camera smoothing -------------------------------------------------------------------------------------
def _hat(w) -> np.ndarray:
    return np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])


def _so3_log(R) -> np.ndarray:
    """Principal axis-angle vector (angle in [0, pi]) of a rotation, through its unit quaternion with w >= 0 (stable near 0 and near pi)."""
    tr = R[0, 0] + R[1, 1] + R[2, 2]
    if tr > 0:
        s = 2.0 * math.sqrt(tr + 1.0)
        q = np.array([(R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s, 0.25 * s])
    else:
        i = int(np.argmax([R[0, 0], R[1, 1], R[2, 2]]))
        j, k = (i + 1) % 3, (i + 2) % 3
        s = 2.0 * math.sqrt(max(1.0 + R[i, i] - R[j, j] - R[k, k], 0.0))
        q = np.zeros(4)
        q[i] = 0.25 * s
        q[j] = (R[j, i] + R[i, j]) / s
        q[k] = (R[k, i] + R[i, k]) / s
        q[3] = (R[k, j] - R[j, k]) / s
    if q[3] < 0:
        q = -q
    q /= np.linalg.norm(q)
    v = q[:3]
    sv = float(np.linalg.norm(v))
    if sv == 0.0:
        return np.zeros(3)
    return v * (2.0 * math.atan2(sv, q[3]) / sv)


def _so3_coeffs(theta: float):
    """A = sin(t)/t, B = (1 - cos(t))/t^2, Cc = (t - sin(t))/t^3, D = (1 - A/(2B))/t^2, with series near 0."""
    t2 = theta * theta
    if theta < 1e-3:
        return 1.0 - t2 / 6.0, 0.5 - t2 / 24.0, 1.0 / 6.0 - t2 / 120.0, 1.0 / 12.0 + t2 / 720.0
    s, c = math.sin(theta), math.cos(theta)
    A, B = s / theta, (1.0 - c) / t2
    return A, B, (theta - s) / (t2 * theta), (1.0 - A / (2.0 * B)) / t2


def _se3_log(M) -> tuple:
    w = _so3_log(M[:3, :3])
    W = _hat(w)
    _, _, _, D = _so3_coeffs(float(np.linalg.norm(w)))
    u = (np.eye(3) - 0.5 * W + D * (W @ W)) @ M[:3, 3]
    return w, u


def _se3_exp(w, u) -> np.ndarray:
    W = _hat(w)
    W2 = W @ W
    A, B, Cc, _ = _so3_coeffs(float(np.linalg.norm(w)))
    out = np.eye(4)
    out[:3, :3] = np.eye(3) + A * W + B * W2
    out[:3, 3] = (np.eye(3) + B * W + Cc * W2) @ u
    return out


def log_space_lerp(begin, end, t) -> np.ndarray:
    """log_space_lerp(A, B, t) = ((B * A^-1).log() * t).exp() * A (common_device.cu:27-36) on 3x4 cameras, returned in float32.

    A restatement, not the reference's arithmetic: the reference evaluates the matrix logarithm and exponential with Eigen's unsupported
    MatrixFunctions module, which is absent from its tree, so its code cannot be executed. Here B * A^-1 is formed in float64 (A inverted as
    a general 4x4 matrix, as the reference does) and its logarithm and the exponential of t times it use the closed-form SE(3) maps: the
    principal rotation vector through the rotation's unit quaternion, so rotations near pi stay accurate, and Rodrigues' formula with its
    translation Jacobian, with series near angle 0. The product with A is float64; one rounding to float32 ends it. For t = 0 the
    exponential is exactly the identity, so the result is A bit for bit, as in the reference. For rigid A and B the rotation part stays
    orthonormal to float32 precision."""
    A = np.eye(4)
    A[:3, :] = np.asarray(begin, f32).reshape(3, 4)
    Bm = np.eye(4)
    Bm[:3, :] = np.asarray(end, f32).reshape(3, 4)
    w, u = _se3_log(Bm @ np.linalg.inv(A))
    t = float(f32(t))
    return (_se3_exp(w * t, u * t) @ A)[:3, :].astype(f32)


def apply_camera_smoothing(state: CameraState, elapsed_ms) -> None:
    """Testbed::apply_camera_smoothing (testbed.cu:2086-2093): decay = powf(0.02f, elapsed_ms / 1000.0f)."""
    if state.camera_smoothing:
        decay = f32(_libm.powf(0.02, float(f32(elapsed_ms) / f32(1000))))
        state.smoothed_camera = log_space_lerp(state.smoothed_camera, state.camera, f32(1) - decay)
    else:
        state.smoothed_camera = np.array(state.camera, f32)


# ---- render_to_cpu ---------------------------------------------------------------------------------------------------------
def sub_frames(path: CameraPath | None, start_time, end_time, fps, spp: int, shutter_fraction, state: CameraState, base_frame: abi.NsbFrame):
    """The spp sub-frames Testbed::render_to_cpu (python_api.cu:129-175) renders, as NsbFrames copied from base_frame (size, boxes, render
    settings): camera0 / camera1 = log_space_lerp(start, end, start_alpha / end_alpha), rolling_shutter 0, spp_index = i, and the focal
    length, focus_z and dof of set_camera_from_time at the sub-frame's mid time (with a path and start_time >= 0; otherwise the state's).
    `state` is updated as the Testbed's members are. Returns (frames, end camera = the new state.smoothed_camera). Without a path (or with
    an empty one) set_camera_from_time leaves the camera as it is, as in the reference. Autofocus is not covered."""
    end_time, start_time, fps, shutter_fraction = f32(end_time), f32(start_time), f32(fps), f32(shutter_fraction)
    if end_time < 0:
        end_time = start_time
    have_path = path is not None and len(path.keyframes) > 0
    start_cam = np.array(state.smoothed_camera, f32)
    if start_time >= 0:
        if have_path:
            state.set_camera_from_keyframe(path.eval_camera_path(end_time))
        apply_camera_smoothing(state, f32(1000) / fps)
    else:
        state.smoothed_camera = np.array(state.camera, f32)
        start_cam = state.smoothed_camera.copy()
    end_cam = np.array(state.smoothed_camera, f32)
    frames = []
    for i in range(spp):
        start_alpha = f32(f32(i) / f32(spp)) * shutter_fraction
        end_alpha = f32(f32(f32(i) + f32(1)) / f32(spp)) * shutter_fraction
        cam0 = log_space_lerp(start_cam, end_cam, start_alpha)
        cam1 = log_space_lerp(start_cam, end_cam, end_alpha)
        if start_time >= 0:
            if have_path:
                mid = start_time + f32(f32(end_time - start_time) * f32(start_alpha + end_alpha)) / f32(2)
                state.set_camera_from_keyframe(path.eval_camera_path(mid))
            state.smoothed_camera = np.array(state.camera, f32)
        f = _frame_from_state(base_frame, state, cam0, cam1)
        for k in range(4):
            f.rolling_shutter[k] = 0.0
        f.spp_index = i
        frames.append(f)
    state.smoothed_camera = end_cam.copy()
    return frames, end_cam


def default_tonemap(linear: bool = True, exposure: float = 0.0) -> abi.NsbTonemap:
    """What render_frame hands CudaRenderBuffer::tonemap by default: m_color_space Linear, m_tonemap_curve Identity, m_exposure,
    m_background_color (0, 0, 0, 1) (testbed.h:502, 765-785), output sRGB unless linear, no clamp."""
    tm = abi.NsbTonemap()
    tm.color_space, tm.tonemap_curve, tm.clamp_output_color = abi.NSB_COLOR_LINEAR, abi.NSB_TONEMAP_IDENTITY, 0
    tm.output_color_space = abi.NSB_COLOR_LINEAR if linear else abi.NSB_COLOR_SRGB
    tm.exposure = float(exposure)
    tm.background_color[:] = [0.0, 0.0, 0.0, 1.0]
    return tm


def render(renderer, base_frame: abi.NsbFrame, path: CameraPath | None, width: int, height: int, spp: int, linear: bool, start_time=-1.0,
           end_time=-1.0, fps=30.0, shutter_fraction=1.0, state: CameraState | None = None, tonemap: abi.NsbTonemap | None = None,
           stream=None) -> np.ndarray:
    """Testbed::render_to_cpu(width, height, spp, linear, start_time, end_time, fps, shutter_fraction): the spp sub-frames in one
    nsb_render_accumulate call; returns the tonemapped frame, float32 [height, width, 4], on the host. tonemap: default_tonemap(linear)
    if None (its output colour space is set from `linear` either way)."""
    state = state if state is not None else CameraState()
    f = abi.NsbFrame.from_buffer_copy(base_frame)
    f.width, f.height = int(width), int(height)
    frames, _ = sub_frames(path, start_time, end_time, fps, spp, shutter_fraction, state, f)
    tm = abi.NsbTonemap.from_buffer_copy(tonemap) if tonemap is not None else default_tonemap(linear)
    tm.output_color_space = abi.NSB_COLOR_LINEAR if linear else abi.NSB_COLOR_SRGB
    import torch

    _, out = renderer.render_accumulate(frames, tm, stream=stream)
    torch.cuda.synchronize(renderer.device)  # the frame may have been rendered on another stream than the copy's
    return out.cpu().numpy()


def initial_state(path: CameraPath, fov_axis: int = 1, zoom: float = 1.0) -> CameraState:
    """A state looking along the path's start: the reference starts the first video frame's shutter at whatever camera the testbed
    held before (m_smoothed_camera); a library caller has none, so this one is the path at t = 0."""
    st = CameraState(fov_axis=fov_axis, zoom=zoom)
    st.set_camera_from_keyframe(path.eval_camera_path(0.0))
    st.smoothed_camera = st.camera.copy()
    return st


def render_video(renderer, base_frame: abi.NsbFrame, path: CameraPath, n_seconds: int, fps: int, spp: int, out_dir: str, smoothing: bool = False,
                 exposure: float = 0.0, state: CameraState | None = None) -> list:
    """scripts/run.py's video loop (run.py:340-356) with PNG files: n = n_seconds * fps frames at base_frame's size, frame i over the
    path times [i/n, (i+1)/n] with shutter 0.5, camera smoothing only for i > 0, linear output, then np.clip(frame * 2**exposure, 0, 1)
    and write_image as 8-bit RGBA on the device (nsb_frame_to_rgba8), written as out_dir/%04d.png. No video is encoded. The copy of frame k
    to the host and its PNG encoding overlap the render of frame k+1 (a side stream and two buffers). Returns the file names."""
    import torch

    state = state if state is not None else initial_state(path)
    n = int(n_seconds) * int(fps)
    W, H = int(base_frame.width), int(base_frame.height)
    os.makedirs(out_dir, exist_ok=True)
    dev = torch.device("cuda", renderer.device)
    render_stream = torch.cuda.current_stream(dev)
    copy_stream = torch.cuda.Stream(dev)
    acc = torch.empty((H, W, 4), dtype=torch.float32, device=dev)
    rgba = torch.empty((H, W, 4), dtype=torch.float32, device=dev)
    px = [torch.empty((H, W, 4), dtype=torch.uint8, device=dev) for _ in range(2)]
    host = [torch.empty((H, W, 4), dtype=torch.uint8, pin_memory=True) for _ in range(2)]
    copied = [None, None]
    tm = default_tonemap(linear=True)
    names = []

    def write(k):
        copied[k & 1].synchronize()
        name = os.path.join(out_dir, "%04d.png" % k)
        slices.write_png(name, host[k & 1].numpy(), 4)
        names.append(name)

    for i in range(n):
        state.camera_smoothing = bool(smoothing) and i > 0
        frames, _ = sub_frames(path, float(i) / n, float(i + 1) / n, fps, spp, 0.5, state, base_frame)  # run.py's times, as pybind rounds them
        slot = i & 1
        if copied[slot] is not None:
            render_stream.wait_event(copied[slot])  # the copy that last read this slot's pixels
        renderer.render_accumulate(frames, tm, accumulate=acc, out=rgba, stream=render_stream.cuda_stream)
        renderer.frame_to_rgba8(rgba, exposure, out=px[slot], stream=render_stream.cuda_stream)
        rendered = torch.cuda.Event()
        rendered.record(render_stream)
        copy_stream.wait_event(rendered)
        with torch.cuda.stream(copy_stream):
            host[slot].copy_(px[slot], non_blocking=True)
        copied[slot] = torch.cuda.Event()
        copied[slot].record(copy_stream)
        if i > 0:
            write(i - 1)
    if n > 0:
        write(n - 1)
    return names
