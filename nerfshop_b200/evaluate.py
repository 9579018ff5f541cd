"""Scores renders against held-out views: the library's version of scripts/run.py --test_transforms and --screenshot_transforms.

  nerf_matrix_to_ngp   <- NerfDataset::nerf_matrix_to_ngp (nerf_loader.h:74-92) in float32, both from_mitsuba branches
  find_image           <- run.py's ground-truth file lookup (run.py:245-256)
  read_image_u8        <- the decode of read_image_imageio (scripts/common.py:132-137): 8-bit RGB or RGBA through PIL
  evaluate             <- run.py's --test_transforms loop (run.py:215-302): ground truth, render and metrics on the device
  screenshots          <- run.py's --screenshot_transforms loop (run.py:309-329), as 8-bit PNG files

The ground truth (nsb_reference_image), the render (nsb_render_accumulate) and the MSE and SSIM of each frame (nsb_image_metrics) stay on
the device; the host decodes the next frame's file meanwhile and reads every frame's two numbers once at the end.
"""
from __future__ import annotations

import json
import os
from dataclasses import dataclass, field

import numpy as np

from . import abi
from . import camera_path as cp
from . import slices

f32 = np.float32


def nerf_matrix_to_ngp(m34, scale: float = 1.0, offset=(0.0, 0.0, 0.0), from_mitsuba: bool = False) -> np.ndarray:
    """NerfDataset::nerf_matrix_to_ngp in float32: the matrix as pybind rounds it, columns 1 and 2 negated, column 3 = col * scale, then
    + offset (each rounded), then from_mitsuba negates columns 0 and 2, otherwise the rows cycle xyz <- yzx. The dataset defaults
    (nerf_loader.h:49-55) are scale 1, offset 0 and from_mitsuba false."""
    r = np.array(np.asarray(m34, np.float64)[:3, :4], f32)
    r[:, 1] = -r[:, 1]
    r[:, 2] = -r[:, 2]
    r[:, 3] = (r[:, 3] * f32(scale)).astype(f32) + np.asarray(offset, f32)
    if from_mitsuba:
        r[:, 0] = -r[:, 0]
        r[:, 2] = -r[:, 2]
        return r
    return r[[1, 2, 0], :].copy()


def find_image(data_dir: str, file_path: str) -> str:
    """run.py's lookup of a frame's ground truth: `.png` appended when the path has no '.', then the path itself, + .png, .jpg, .jpeg
    and, last, + .exr (returned even when it does not exist, as run.py does; read_image_u8 then fails)."""
    p = file_path if "." in file_path else file_path + ".png"
    for cand in (p, p + ".png", p + ".jpg", p + ".jpeg"):
        name = os.path.join(data_dir, cand)
        if os.path.isfile(name):
            return name
    return os.path.join(data_dir, p + ".exr")


def read_image_u8(path: str) -> np.ndarray:
    """The 8-bit pixels imageio hands read_image for a PNG or JPEG (through Pillow): uint8 [H, W, 3 or 4]. Grayscale, palette-free
    16-bit, and every other mode or format (.exr, .bin) raise ValueError."""
    if os.path.splitext(path)[1].lower() in (".exr", ".bin"):
        raise ValueError(f"{path}: .exr and .bin ground truth is not supported (8-bit PNG or JPEG only)")
    if not os.path.isfile(path):
        raise FileNotFoundError(path)
    from PIL import Image

    with Image.open(path) as im:
        if im.mode == "P":  # palette PNGs: imageio expands them to RGB or RGBA
            im = im.convert("RGBA" if "transparency" in im.info else "RGB")
        if im.mode not in ("RGB", "RGBA"):
            raise ValueError(f"{path}: mode {im.mode} is not 8-bit RGB or RGBA (grayscale and 16-bit images are not supported)")
        return np.array(im, dtype=np.uint8)


def load_transforms(path: str) -> dict:
    with open(path) as fh:
        return json.load(fh)


def mse2psnr(x: float) -> float:
    """common.py:49 in float64; MSE 0 gives inf."""
    with np.errstate(divide="ignore"):
        return float(-10.0 * np.log(x) / np.log(10.0))


def test_frame(base_frame: abi.NsbFrame, srgb: bool = False) -> abi.NsbFrame:
    """base_frame with run.py's evaluation settings: snap_to_pixel_centers, rendering_min_transmittance 1e-4, and with srgb (its
    --nerf_compatibility) cone_angle_constant 0."""
    f = abi.NsbFrame.from_buffer_copy(base_frame)
    f.snap_to_pixel_centers = 1
    f.min_transmittance = 1e-4
    if srgb:
        f.cone_angle_constant = 0.0
    return f


def _tonemap(srgb: bool) -> abi.NsbTonemap:
    """render_to_cpu's tonemap with linear output, background (0, 0, 0, 1) and the colour space sRGB with srgb (run.py sets
    testbed.color_space with --nerf_compatibility)."""
    tm = cp.default_tonemap(linear=True)
    if srgb:
        tm.color_space = abi.NSB_COLOR_SRGB
    return tm


def _camera_state(camera_angle_x: float, m34, dataset) -> cp.CameraState:
    """testbed.fov_axis = 0, testbed.fov = camera_angle_x * 180 / pi (set_fov), set_nerf_camera_matrix(m34)."""
    st = cp.CameraState(fov_axis=0)
    st.relative_focal_length = np.full(2, cp.fov_to_focal_length(1, float(camera_angle_x) * 180 / np.pi), f32)
    st.camera = nerf_matrix_to_ngp(m34, *dataset)
    return st


def sub_frames(base_frame: abi.NsbFrame, width: int, height: int, spp: int, state: cp.CameraState) -> list:
    """testbed.render(width, height, spp, True)'s sub-frames: render_to_cpu with start_time -1 (camera_path.sub_frames)."""
    f = abi.NsbFrame.from_buffer_copy(base_frame)
    f.width, f.height = int(width), int(height)
    frames, _ = cp.sub_frames(None, -1.0, -1.0, 30.0, spp, 1.0, state, f)
    return frames


@dataclass
class EvalResult:
    """Per-frame numbers and run.py's summary values (run.py:286-302)."""
    files: list = field(default_factory=list)
    mse: list = field(default_factory=list)     # float(compute_error("MSE", A, R)) per frame
    ssim: list = field(default_factory=list)
    psnr: list = field(default_factory=list)    # mse2psnr(mse)
    mean_psnr: float = 0.0
    min_psnr: float = 1000.0
    max_psnr: float = 0.0
    mean_ssim: float = 0.0
    psnr_avgmse: float = 0.0

    def summary(self) -> str:
        """The line run.py prints."""
        return f"PSNR={self.mean_psnr} [min={self.min_psnr} max={self.max_psnr}] SSIM={self.mean_ssim}"


def evaluate(renderer, base_frame: abi.NsbFrame, transforms, spp: int = 8, srgb: bool = False, out_dir: str | None = None,
             dataset=(1.0, (0.0, 0.0, 0.0), False)) -> EvalResult:
    """run.py's --test_transforms loop. transforms: the path of a NeRF-style transforms.json (its directory is the data directory).
    base_frame: the scene's frame settings (boxes, activations, operators); test_frame's settings are applied to it, each frame takes
    its ground truth's size. dataset: (scale, offset, from_mitsuba) of the snapshot (snapshot.load_dataset_transform). srgb: run.py's
    --nerf_compatibility (colour space sRGB with its ground-truth blend, cone angle 0). With out_dir, frame 0's ref.png, out.png and
    diff.png are written there as run.py writes them. RGB ground truth gets alpha 1."""
    import torch

    tj = load_transforms(transforms)
    data_dir = os.path.dirname(transforms)
    frames_j = tj["frames"]
    base = test_frame(base_frame, srgb)
    tm = _tonemap(srgb)
    bg = [float(v) for v in tm.background_color]
    dev = torch.device("cuda", renderer.device)
    stream = torch.cuda.current_stream(dev)
    results = torch.zeros((len(frames_j), 2), dtype=torch.float32, device=dev)
    res = EvalResult()
    first = None
    for i, fj in enumerate(frames_j):
        name = find_image(data_dir, fj["file_path"])
        px = read_image_u8(name)  # overlaps the device work queued for frame i - 1
        res.files.append(name)
        H, W = px.shape[0], px.shape[1]
        px_dev = torch.from_numpy(px).pin_memory().to(dev, non_blocking=True)  # torch's pinned pool keeps the block until the copy is done
        ref = renderer.reference_image(px_dev, srgb_blend=srgb and px.shape[2] == 4, background=bg, stream=stream.cuda_stream)
        st = _camera_state(tj["camera_angle_x"], np.asarray(fj["transform_matrix"], np.float64)[:-1, :], dataset)
        _, image = renderer.render_accumulate(sub_frames(base, W, H, spp, st), tm, stream=stream.cuda_stream)
        renderer.image_metrics(image, ref, out=results[i], stream=stream.cuda_stream)
        if i == 0 and out_dir:
            first = (image, ref)
    if first is not None:
        _write_first(renderer, out_dir, *first, stream)
    host = results.cpu().numpy()  # the one synchronisation
    totmse = totpsnr = totssim = 0.0
    for i in range(len(frames_j)):
        mse, ssim = float(host[i, 0]), float(host[i, 1])
        psnr = mse2psnr(mse)
        res.mse.append(mse)
        res.ssim.append(ssim)
        res.psnr.append(psnr)
        totmse += mse
        totpsnr += psnr
        totssim += ssim
        res.min_psnr = psnr if psnr < res.min_psnr else res.min_psnr
        res.max_psnr = psnr if psnr > res.max_psnr else res.max_psnr
    n = len(frames_j) or 1
    res.psnr_avgmse = mse2psnr(totmse / n)
    res.mean_psnr = totpsnr / n
    res.mean_ssim = totssim / n
    return res


def _write_first(renderer, out_dir: str, image, ref, stream) -> None:
    """run.py's ref.png, out.png and diff.png of frame 0: write_image of the ground truth, the render and |image - ref| with alpha 1, the
    8-bit pixels from nsb_frame_to_rgba8."""
    import torch

    os.makedirs(out_dir, exist_ok=True)
    diff = (image - ref).abs()
    diff[..., 3] = 1.0
    for fname, img in (("ref.png", ref), ("out.png", image), ("diff.png", diff)):
        px = renderer.frame_to_rgba8(img.contiguous(), 0.0, stream=stream.cuda_stream)
        slices.write_png(os.path.join(out_dir, fname), px.cpu().numpy(), 4)
    torch.cuda.synchronize(renderer.device)


def screenshot_name(screenshot_dir: str, file_path: str) -> str:
    """run.py's output name: the frame's basename in screenshot_dir, + .png when it has no extension."""
    out = os.path.join(screenshot_dir, os.path.basename(file_path))
    if not os.path.splitext(out)[1]:
        out = out + ".png"
    return out


def screenshots(renderer, base_frame: abi.NsbFrame, transforms, screenshot_dir: str, frames=None, spp: int = 16, width: int = 0, height: int = 0,
                dataset=(1.0, (0.0, 0.0, 0.0), False)) -> list:
    """run.py's --screenshot_transforms loop: for each index in frames (all if None), the camera of that view (fov_axis 0, the fov from
    camera_angle_x), rendered at width x height (0: the file's w / h) with spp samples and linear output, written as write_image would
    write an 8-bit PNG (nsb_frame_to_rgba8 with exposure 0). base_frame's settings are used as they are. Returns the file names. Only
    PNG output is written: a name with another extension raises ValueError before anything is rendered."""
    tj = load_transforms(transforms)
    idx = range(len(tj["frames"])) if not frames else [int(k) for k in frames]
    jobs = []
    for k in idx:
        fj = tj["frames"][k]
        name = screenshot_name(screenshot_dir, fj["file_path"])
        if os.path.splitext(name)[1].lower() != ".png":
            raise ValueError(f"{name}: screenshots are written as PNG files only")
        jobs.append((fj, name))
    tm = _tonemap(False)
    W, H = int(width or int(tj["w"])), int(height or int(tj["h"]))
    names = []
    for fj, name in jobs:
        st = _camera_state(tj["camera_angle_x"], np.asarray(fj["transform_matrix"], np.float64)[:-1, :], dataset)
        _, image = renderer.render_accumulate(sub_frames(base_frame, W, H, spp, st), tm)
        px = renderer.frame_to_rgba8(image, 0.0)
        d = os.path.dirname(name)
        if d:
            os.makedirs(d, exist_ok=True)
        slices.write_png(name, px.cpu().numpy(), 4)
        names.append(name)
    return names
