"""Times one 1920x1080 video frame at spp 8 on the synthetic fox-config scene along a 3-keyframe orbit path, per output frame:
  - nsb_render_accumulate (one call: 8 sub-frames rendered, accumulated, one tonemap) against the same work as a Python loop of the existing
    calls (zero the frame and depth buffers, NerfRenderer.render, NerfRenderer.accumulate per sub-frame, then NerfRenderer.tonemap), CUDA
    events around the whole frame and the host wall clock of the calls (the enqueue); both outputs are compared bit for bit first;
  - nsb_frame_to_rgba8 (CUDA events over 50 calls);
  - the device-to-host copy into pinned memory of the 8-bit RGBA frame (8.3 MB) and of the float4 frame (33.2 MB);
  - the PNG encoding on the host (nerfshop_b200.slices.write_png, one thread, zlib level 6; wall clock).
The card, its power limit and SM clock are read in the same run.
  python tools/profile_video.py [--frames N]"""
import argparse
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from nerfshop_b200 import camera_path as cp  # noqa: E402
from nerfshop_b200 import slices  # noqa: E402
from nerfshop_b200 import synthetic as syn  # noqa: E402
from nerfshop_b200.renderer import NerfRenderer  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--frames", type=int, default=12, help="video frames timed per measurement (after one warm-up frame)")
ap.add_argument("--width", type=int, default=1920)
ap.add_argument("--height", type=int, default=1080)
ap.add_argument("--spp", type=int, default=8)
args = ap.parse_args()
W, H, SPP = args.width, args.height, args.spp

print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
model = syn.make_model(seed=1337)
occ = syn.make_occupancy(model)
r = NerfRenderer(0)
r.upload_model(model.desc, model.params)
r.upload_occupancy(occ)
cams = syn.orbit_cameras(120)
path = cp.CameraPath([cp.CameraKeyframe.from_matrix(cams[i]) for i in (10, 20, 30)])
base = syn.make_frame(model, cams[10], W, H)
tm = cp.default_tonemap(linear=True)
n_video = args.frames + 1
state = cp.initial_state(path)
videos = []
for i in range(n_video):
    state.camera_smoothing = i > 0
    videos.append(cp.sub_frames(path, i / n_video, (i + 1) / n_video, 30, SPP, 0.5, state, base)[0])

acc = torch.empty((H, W, 4), device="cuda")
out = torch.empty_like(acc)
fb = torch.empty_like(acc)
depth = torch.empty((H, W), device="cuda")
acc2 = torch.empty_like(acc)


def one_call(frames):
    r.render_accumulate(frames, tm, accumulate=acc, out=out)
    return out


def python_loop(frames):
    for f in frames:
        fb.zero_()
        depth.zero_()
        r.render(f, fb, depth)
        r.accumulate(fb, acc2, f.spp_index, tm.color_space)
    return r.tonemap(acc2, tm)


def timed_frames(fn):
    dev_ms, host_ms = [], []
    for k, frames in enumerate(videos):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        t0 = time.perf_counter()
        fn(frames)
        t1 = time.perf_counter()
        e1.record()
        torch.cuda.synchronize()
        if k > 0:  # frame 0 warms up
            dev_ms.append(e0.elapsed_time(e1))
            host_ms.append((t1 - t0) * 1e3)
    return float(np.median(dev_ms)), float(np.median(host_ms))


# same bits first
a = one_call(videos[0]).clone()
b = python_loop(videos[0])
torch.cuda.synchronize()
same = bool(torch.equal(a.view(torch.int32), b.view(torch.int32)))
print(f"render_accumulate == python loop, bit for bit: {same}")
assert same
for rep in range(2):  # alternate the two, twice, to see the spread
    d1, h1 = timed_frames(one_call)
    d2, h2 = timed_frames(python_loop)
    print(f"[{rep}] {W}x{H} spp {SPP}, per output frame (median of {args.frames}): nsb_render_accumulate {d1:.2f} ms device, {h1:.3f} ms enqueue | "
          f"python loop of existing calls {d2:.2f} ms device, {h2:.3f} ms enqueue")

px = torch.empty((H, W, 4), dtype=torch.uint8, device="cuda")
r.frame_to_rgba8(out, 0.0, out=px)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
torch.cuda.synchronize()
e0.record()
for _ in range(50):
    r.frame_to_rgba8(out, 0.0, out=px)
e1.record()
torch.cuda.synchronize()
print(f"nsb_frame_to_rgba8: {e0.elapsed_time(e1) / 50 * 1e3:.1f} us per frame ({W * H * 20 / (e0.elapsed_time(e1) / 50 * 1e-3) / 1e9:.0f} GB/s of 16 B read + 4 B written per pixel)")

host8 = torch.empty((H, W, 4), dtype=torch.uint8, pin_memory=True)
host32 = torch.empty((H, W, 4), dtype=torch.float32, pin_memory=True)
for name, src, dst in (("8-bit RGBA", px, host8), ("float4", out, host32)):
    ms = []
    for _ in range(21):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        dst.copy_(src, non_blocking=True)
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    mb = src.numel() * src.element_size() / 1e6
    print(f"D2H {name} ({mb:.1f} MB, pinned): {np.median(ms[1:]):.3f} ms ({mb / np.median(ms[1:]):.1f} GB/s)")

pixels = host8.numpy()
with tempfile.TemporaryDirectory() as d:
    ms = []
    for k in range(5):
        t0 = time.perf_counter()
        slices.write_png(os.path.join(d, "%04d.png" % k), pixels, 4)
        ms.append((time.perf_counter() - t0) * 1e3)
    size = os.path.getsize(os.path.join(d, "0000.png"))
print(f"PNG encoding on the host (write_png, one thread, zlib 6): {np.median(ms):.1f} ms per frame ({size / 1e6:.2f} MB file)")

with tempfile.TemporaryDirectory() as d:
    t0 = time.perf_counter()
    cp.render_video(r, base, path, n_seconds=1, fps=n_video, spp=SPP, out_dir=d)
    dt = (time.perf_counter() - t0) * 1e3
print(f"render_video end to end: {n_video} frames in {dt:.0f} ms ({dt / n_video:.1f} ms per frame, copies and PNG encoding overlapped with rendering)")
r.close()
