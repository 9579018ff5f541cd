"""Times the image-quality metrics on the GPU: nsb_reference_image + nsb_image_metrics per frame (CUDA events, as effective GB/s of the
bytes they must read and write), run.py's numpy metric block on this host for the same frames, and evaluate's time per test view at
800x800 and 8 spp against the reference's structure (render_to_cpu into host memory, then the numpy block).

  python tools/profile_evaluate.py [--reps 20]     prints one JSON line with the card, its power limit and max SM clock"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from scipy.ndimage import convolve1d  # noqa: E402

import eval_rule as er  # noqa: E402
from nerfshop_b200 import camera_path as cp  # noqa: E402
from nerfshop_b200 import evaluate as ev  # noqa: E402
from nerfshop_b200 import slices  # noqa: E402
from nerfshop_b200 import synthetic as syn  # noqa: E402
from nerfshop_b200.renderer import NerfRenderer  # noqa: E402


def numpy_block(image, ref):
    """run.py:286-290 with scripts/common.py's linear_to_srgb, compute_error("MSE") and compute_error("SSIM"), transcribed: numpy and
    scipy on one host thread."""
    def l2s(img):
        return np.where(img > 0.0031308, 1.055 * (img ** (1.0 / 2.4)) - 0.055, 12.92 * img)

    def lum(a):
        a = np.maximum(0, a) ** 0.4545454545
        return 0.2126 * a[:, :, 0] + 0.7152 * a[:, :, 1] + 0.0722 * a[:, :, 2]

    def blur(a):
        return convolve1d(convolve1d(a, er.K, axis=0), er.K, axis=1)

    with np.errstate(all="ignore"):
        A = np.clip(l2s(image[..., :3]), 0.0, 1.0)
        R = np.clip(l2s(ref[..., :3]), 0.0, 1.0)
        A[np.logical_not(np.isfinite(A))] = 0
        A = np.maximum(A, 0.0)
        m = (A - R) ** 2
        m[np.logical_not(np.isfinite(m))] = 0
        mse = np.mean(np.mean(m, axis=2))
        a, b = lum(np.clip(A, 0.0, 1.0)), lum(np.clip(R, 0.0, 1.0))
        mA, mB = blur(a), blur(b)
        sA, sB, sAB = blur(a * a) - mA ** 2, blur(b * b) - mB ** 2, blur(a * b) - mA * mB
        e = ((2.0 * mA * mB + 0.01 ** 2) / (mA * mA + mB * mB + 0.01 ** 2)) * ((2.0 * sAB + 0.03 ** 2) / (sA + sB + 0.03 ** 2))
        e[np.logical_not(np.isfinite(e))] = 0
    return float(mse), float(np.mean(e))


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    r = NerfRenderer(0)
    model = syn.make_model(seed=1337)
    r.upload_model(model.desc, model.params)
    r.upload_occupancy(syn.make_occupancy(model))
    out = {"card": _card()}
    for H, W in ((800, 800), (1080, 1920)):
        rng = np.random.default_rng(0)
        px = torch.from_numpy(rng.integers(0, 256, (H, W, 4), dtype=np.uint8)).cuda()
        img = torch.rand((H, W, 4), device="cuda")
        res = torch.empty(2, device="cuda")
        for _ in range(3):
            ref = r.reference_image(px)
            r.image_metrics(img, ref, out=res)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            r.reference_image(px, out=ref)
            r.image_metrics(img, ref, out=res)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.reps
        nbytes = H * W * (4 + 16 + 16 + 16 + 8 + 8)  # bytes in, GT out, both frames in, both maps written and read back
        t = time.perf_counter()
        numpy_block(img.cpu().numpy(), ref.cpu().numpy())
        host_ms = (time.perf_counter() - t) * 1e3
        out[f"{H}x{W}"] = {"device_ms": round(ms, 4), "effective_GBps": round(nbytes / ms / 1e6, 1), "numpy_block_host_ms": round(host_ms, 1)}
    with tempfile.TemporaryDirectory() as d:
        os.makedirs(os.path.join(d, "test"))
        cams = syn.orbit_cameras(120)
        base = syn.make_frame(model, np.eye(3, 4, dtype=np.float32), 800, 800)
        frames = []
        for i in range(8):
            nerf = np.asarray(cams[i * 15], np.float64)[[2, 0, 1], :]  # the inverse of nerf_matrix_to_ngp with the dataset defaults
            nerf[:, 1] *= -1
            nerf[:, 2] *= -1
            nerf = np.vstack([nerf[:, :4], [0, 0, 0, 1]])
            slices.write_png(os.path.join(d, "test", f"r_{i}.png"), np.random.default_rng(i).integers(0, 256, (800, 800, 4), dtype=np.uint8), 4)
            frames.append({"file_path": f"./test/r_{i}", "transform_matrix": nerf.tolist()})
        tr = os.path.join(d, "transforms_test.json")
        json.dump({"camera_angle_x": 0.69, "frames": frames}, open(tr, "w"))
        ev.evaluate(r, base, tr)
        torch.cuda.synchronize()
        t = time.perf_counter()
        ev.evaluate(r, base, tr)
        torch.cuda.synchronize()
        out["evaluate_ms_per_view_800x800_8spp"] = round((time.perf_counter() - t) * 1e3 / len(frames), 2)
        t = time.perf_counter()
        tj = json.load(open(tr))
        for fj in tj["frames"]:  # the reference's structure: render_to_cpu, then read_image and the numpy block on the host
            st = ev._camera_state(0.69, np.asarray(fj["transform_matrix"])[:-1, :], (1.0, (0.0, 0.0, 0.0), False))
            image = cp.render(r, ev.test_frame(base), None, 800, 800, 8, True, state=st, tonemap=ev._tonemap(False))
            refi = er.reference_image(ev.read_image_u8(ev.find_image(d, fj["file_path"])), pw=er.pow_np)
            numpy_block(image, refi)
        out["host_metrics_structure_ms_per_view_800x800_8spp"] = round((time.perf_counter() - t) * 1e3 / len(frames), 2)
    print(json.dumps(out))
    r.close()


if __name__ == "__main__":
    main()
