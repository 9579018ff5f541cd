"""Image-quality metrics on the GPU (ABI 9): nsb_reference_image and nsb_image_metrics against the host restatement (tests/eval_rule.py)
and numpy/scipy's own chain, the device pows against correctly rounded float32 pow, and nerfshop_b200.evaluate's test-view scores and
screenshots against a transcription of run.py's loops built on the existing calls."""
import atexit
import ctypes as C
import json
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest
from scipy.ndimage import convolve1d

import edit_fixtures as fx
import eval_rule as er
from nerfshop_b200 import abi
from nerfshop_b200 import build as nsb_build
from nerfshop_b200 import camera_path as cp
from nerfshop_b200 import evaluate as ev
from nerfshop_b200 import slices, snapshot
from nerfshop_b200 import synthetic as syn
from png_decode import decode_png
from test_gpu_camera_path import _check_bytes

pytestmark = pytest.mark.gpu
F32 = np.float32
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "nerfshop_b200", "csrc")

# the device functions of nsb_eval.cuh on their own: the pows, A / R and both luminances per pixel
_PROBE_SRC = r"""
#include <cstdint>
#include <cuda_runtime.h>
#include "nsb_eval.cuh"
__global__ void k_pow(uint32_t n, int kind, const float* x, float* y) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const float v = x[i];
	y[i] = kind == 0 ? evalm::pow_cr(v, (float)(1.0 / 2.4)) : kind == 1 ? evalm::pow_cr(v, (float)2.4) : kind == 2 ? evalm::pow_cr(v, (float)0.4545454545)
	     : kind == 3 ? evalm::linear_to_srgb(v) : evalm::srgb_to_linear(v);
}
__global__ void k_color(uint32_t n, const float4* img, const float4* ref, float* A, float* R, float* la, float* lb) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const float4 v = img[i], w = ref[i];
	const float a[3] = {evalm::metric_a(v.x), evalm::metric_a(v.y), evalm::metric_a(v.z)};
	const float r[3] = {evalm::metric_r(w.x), evalm::metric_r(w.y), evalm::metric_r(w.z)};
	for (int k = 0; k < 3; ++k) A[3 * i + k] = a[k], R[3 * i + k] = r[k];
	la[i] = evalm::lum_of(a);
	lb[i] = evalm::lum_of(r);
}
extern "C" int probe_pow(uint32_t n, int kind, const float* x_dev, float* y_dev) {
	k_pow<<<(n + 255) / 256, 256>>>(n, kind, x_dev, y_dev);
	return cudaDeviceSynchronize() == cudaSuccess ? 0 : 1;
}
extern "C" int probe_color(uint32_t n, const float* img, const float* ref, float* A, float* R, float* la, float* lb) {
	k_color<<<(n + 255) / 256, 256>>>(n, (const float4*)img, (const float4*)ref, A, R, la, lb);
	return cudaDeviceSynchronize() == cudaSuccess ? 0 : 1;
}
"""
_probe = None


def probe() -> C.CDLL:
    """The probe, compiled into a temporary directory with the product's nvcc flags."""
    global _probe
    if _probe is None:
        tmp = tempfile.mkdtemp(prefix="nsb_eval_probe_")
        atexit.register(shutil.rmtree, tmp, True)
        src, lib = os.path.join(tmp, "probe.cu"), os.path.join(tmp, "libprobe.so")
        with open(src, "w") as fh:
            fh.write(_PROBE_SRC)
        ccbin = ["-ccbin", "/usr/bin/g++"] if os.path.exists("/usr/bin/g++") else []
        res = subprocess.run([nsb_build._nvcc()] + nsb_build.NVCC_FLAGS + ccbin + ["-I", CSRC, "-o", lib, src], capture_output=True, text=True)
        assert res.returncode == 0, res.stdout + res.stderr
        l = C.CDLL(lib)
        l.probe_pow.argtypes = [C.c_uint32, C.c_int, C.c_void_p, C.c_void_p]
        l.probe_color.argtypes = [C.c_uint32] + [C.c_void_p] * 6
        _probe = l
    return _probe


def _same(a, b) -> bool:
    return np.array_equal(np.asarray(a, F32).view(np.uint32), np.asarray(b, F32).view(np.uint32))


def _dev_pow(x, kind):
    import torch

    xd = torch.from_numpy(np.ascontiguousarray(x, F32)).cuda()
    yd = torch.empty_like(xd)
    assert probe().probe_pow(xd.numel(), kind, xd.data_ptr(), yd.data_ptr()) == 0
    return yd.cpu().numpy()


# ---- nsb_reference_image ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("srgb_blend", [False, True])
def test_reference_image_every_byte_pair(renderer, srgb_blend):
    import torch

    v, a = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    px = np.stack([v, (v + 85) % 256, (v + 170) % 256, a], -1).astype(np.uint8)  # every (value, alpha) pair in each colour channel
    bg = (0.25, 0.5, 0.75, 1.0)
    got = renderer.reference_image(torch.from_numpy(px).cuda(), srgb_blend=srgb_blend, background=bg).cpu().numpy()
    assert _same(got, er.reference_image(px, srgb_blend, bg))
    d = er.ulps(got, er.reference_image(px, srgb_blend, bg, er.pow_np))
    print(f"reference_image srgb_blend={srgb_blend}: {int((d > 0).sum())} of {d.size} values differ from numpy's own chain, max {int(d.max())} ulp")
    rgb = np.stack([np.arange(256)] * 3, -1).astype(np.uint8).reshape(16, 16, 3)
    got = renderer.reference_image(torch.from_numpy(rgb).cuda(), srgb_blend=srgb_blend, background=bg).cpu().numpy()
    assert _same(got, er.reference_image(rgb, False))  # the blend is for RGBA only


def _same_nan(a, b) -> bool:
    """Bit for bit, every NaN counting as one value (the GPU's NaN is canonical; numpy keeps the input's bits)."""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and _same(a[~na], b[~nb])


def test_device_pows_every_float_in_unit_interval():
    """Every float32 in [0, 1] through each pow: the device's float64 pow rounded once equals correctly rounded float32 pow except where
    the exact power lies within 2^-40 (relative) of a float32 rounding boundary, closer than float64 pow's own error; those values are
    counted and differ by 1 ulp. Plus the two sRGB branch points and 8 ulps on each side."""
    top = int(np.array(1.0, F32).view(np.uint32))
    chunk = 1 << 25
    ties = 0
    for kind, y in enumerate((F32(1.0 / 2.4), F32(2.4), er.GAMMA)):
        for lo in range(0, top + 1, chunk):
            x = np.arange(lo, min(lo + chunk, top + 1), dtype=np.uint32).view(F32)
            got = _dev_pow(x, kind)
            with np.errstate(all="ignore"):
                fast = np.power(x.astype(np.float64), np.float64(y)).astype(F32)  # pow_cr without its tie check
            idx = np.nonzero(got.view(np.uint32) != fast.view(np.uint32))[0]
            want = er.pow_cr(x[idx], y)  # settles the few values whose float64 pows round apart
            bad = got[idx].view(np.uint32) != want.view(np.uint32)
            if bad.any():
                g, w, xb = got[idx][bad], want[bad], x[idx][bad]
                assert (er.ulps(g, w) == 1).all(), (kind, xb[:8])
                mid = (g.astype(np.float64) + w.astype(np.float64)) / 2
                exact = np.array([float(er._exact_pow(float(v), float(y))) for v in xb])
                assert (np.abs(exact - mid) <= mid * 2.0 ** -40).all(), (kind, xb[:8])
                ties += int(bad.sum())
                print(f"pow kind {kind}: {int(bad.sum())} near-tie value(s), e.g. x = {float(xb[0])!r}")
    print(f"device pows: {ties} of {3 * (top + 1)} values round a near-tie the other way")
    assert ties <= 16
    for kind, lim, fn in ((3, F32(0.0031308), er.linear_to_srgb), (4, F32(0.04045), er.srgb_to_linear)):
        steps = [lim]
        up = dn = lim
        for _ in range(8):
            up, dn = np.nextafter(up, F32(1)), np.nextafter(dn, F32(0))
            steps += [up, dn]
        x = np.array(steps, F32)
        assert _same(_dev_pow(x, kind), fn(x))


# ---- nsb_image_metrics --------------------------------------------------------------------------------------------------
SHAPES = [(1, 1), (1, 7), (7, 1), (2, 2), (3, 5), (64, 64), (333, 517), (800, 800), (1080, 1920), (1920, 1080)]


def _inputs(H, W, seed):
    rng = np.random.default_rng(seed)
    ref = rng.random((H, W, 4), dtype=F32)
    img = (ref + F32(0.05) * rng.standard_normal((H, W, 4)).astype(F32)).astype(F32)
    n = H * W
    k = max(1, n // 50)
    special = np.array([np.nan, np.inf, -np.inf, 1e4, 37.5, -1.0, -0.0, 0.0, 0.0031308, 0.04045,
                        np.nextafter(F32(0.0031308), F32(1)), np.nextafter(F32(0.0031308), F32(0))], F32)
    img.reshape(-1, 4)[rng.integers(0, n, k), rng.integers(0, 4, k)] = rng.choice(special, k)
    ref.reshape(-1, 4)[rng.integers(0, n, k), 3] = 0.0  # alpha 0
    ref.reshape(-1, 4)[rng.integers(0, n, max(1, k // 4)), rng.integers(0, 3, max(1, k // 4))] = rng.choice(special, max(1, k // 4))
    return img, ref


def _scipy_rest(A, R, la, lb):
    """run.py / common.py's chain after A, R and the luminances, with numpy and scipy themselves."""
    def blur(a):
        return convolve1d(convolve1d(a, er.K, axis=0), er.K, axis=1)

    with np.errstate(all="ignore"):
        m = (A - R) ** 2
        m[np.logical_not(np.isfinite(m))] = 0
        mm = np.mean(m, axis=2)
        mA, mB = blur(la), blur(lb)
        sA, sB, sAB = blur(la * la) - mA ** 2, blur(lb * lb) - mB ** 2, blur(la * lb) - mA * mB
        e = ((2.0 * mA * mB + 0.01 ** 2) / (mA * mA + mB * mB + 0.01 ** 2)) * ((2.0 * sAB + 0.03 ** 2) / (sA + sB + 0.03 ** 2))
        e[np.logical_not(np.isfinite(e))] = 0
    return mm, e, np.mean(mm), np.mean(e)


@pytest.mark.parametrize("shape", SHAPES, ids=[f"{h}x{w}" for h, w in SHAPES])
def test_image_metrics(renderer, shape):
    import torch

    H, W = shape
    img, ref = _inputs(H, W, H * 7919 + W)
    di, dr = torch.from_numpy(img).cuda(), torch.from_numpy(ref).cuda()
    mm_d = torch.empty((H, W), dtype=torch.float32, device="cuda")
    sm_d = torch.empty_like(mm_d)
    out = renderer.image_metrics(di, dr, mse_map=mm_d, ssim_map=sm_d)
    out2 = renderer.image_metrics(di, dr)  # the context's own maps
    n = H * W
    A, R = torch.empty((H, W, 3), device="cuda"), torch.empty((H, W, 3), device="cuda")
    la, lb = torch.empty((H, W), device="cuda"), torch.empty((H, W), device="cuda")
    assert probe().probe_color(n, di.data_ptr(), dr.data_ptr(), A.data_ptr(), R.data_ptr(), la.data_ptr(), lb.data_ptr()) == 0
    A, R, la, lb = (t.cpu().numpy() for t in (A, R, la, lb))
    got = out.cpu().numpy()
    mm, sm = mm_d.cpu().numpy(), sm_d.cpu().numpy()
    assert _same(got, out2.cpu().numpy())
    w_mm, w_sm, w_mse, w_ssim = _scipy_rest(A, R, la, lb)
    assert _same(mm, w_mm) and _same(sm, w_sm)
    assert _same(got, [w_mse, w_ssim])
    assert _same(got, [np.mean(mm), np.mean(sm)])
    # the pow stages against the correctly rounded restatement
    assert _same(A, er.metric_a(img[..., :3])) and _same_nan(R, er.metric_r(ref[..., :3]))
    assert _same(la, er.luminance(A)) and _same_nan(lb, er.luminance(R))
    full = er.metrics(img, ref, er.pow_np)  # run.py's whole chain with numpy's pow
    print(f"{H}x{W}: vs numpy's pow |dPSNR| {abs(ev.mse2psnr(float(got[0])) - ev.mse2psnr(float(full['mse']))):.3g}, "
          f"|dSSIM| {abs(float(got[1]) - float(full['ssim'])):.3g}")
    clean = torch.from_numpy(np.random.default_rng(H + W).random((H, W, 4), dtype=F32)).cuda()  # finite colours: no pixel's SSIM is zeroed
    same = renderer.image_metrics(clean, clean).cpu().numpy()
    assert same[0] == 0.0 and same[1] == 1.0


def test_metrics_argument_errors_write_nothing(renderer):
    import torch

    lib, ctx = renderer.lib, renderer.ctx
    img = torch.rand((8, 8, 4), device="cuda")
    px = torch.zeros((8, 8, 4), dtype=torch.uint8, device="cuda")
    out = torch.full((8, 8, 4), 7.0, device="cuda")
    res = torch.full((2,), 7.0, device="cuda")
    bg = (C.c_float * 4)(0, 0, 0, 1)
    E = abi.NSB_ERR_INVALID
    for args in [(None, px.data_ptr(), 8, 8, 4, 0, bg, out.data_ptr()), (ctx, None, 8, 8, 4, 0, bg, out.data_ptr()), (ctx, px.data_ptr(), 8, 8, 4, 0, bg, None),
                 (ctx, px.data_ptr(), 0, 8, 4, 0, bg, out.data_ptr()), (ctx, px.data_ptr(), 8, -1, 4, 0, bg, out.data_ptr()),
                 (ctx, px.data_ptr(), 8, 8, 2, 0, bg, out.data_ptr()), (ctx, px.data_ptr(), 8, 8, 5, 0, bg, out.data_ptr()),
                 (ctx, px.data_ptr(), 8, 8, 4, 1, None, out.data_ptr()), (ctx, px.data_ptr(), 8, 8, 4, 2, bg, out.data_ptr())]:
        assert lib.nsb_reference_image(*args, None) == E
    for args in [(None, img.data_ptr(), img.data_ptr(), 8, 8, res.data_ptr()), (ctx, None, img.data_ptr(), 8, 8, res.data_ptr()),
                 (ctx, img.data_ptr(), None, 8, 8, res.data_ptr()), (ctx, img.data_ptr(), img.data_ptr(), 8, 8, None),
                 (ctx, img.data_ptr(), img.data_ptr(), 0, 8, res.data_ptr()), (ctx, img.data_ptr(), img.data_ptr(), 8, -3, res.data_ptr()),
                 (ctx, img.data_ptr() + 4, img.data_ptr(), 8, 8, res.data_ptr())]:
        assert lib.nsb_image_metrics(*args, None, None, None) == E
    torch.cuda.synchronize()
    assert bool((out == 7.0).all()) and bool((res == 7.0).all())


# ---- evaluate and screenshots end to end ----------------------------------------------------------------------------------
GW, GH, CAX = 96, 72, 0.69


def ngp_matrix_to_nerf(m, scale, offset, from_mitsuba=False) -> np.ndarray:
    """The inverse of nerf_matrix_to_ngp, float64, as a 4x4 transform_matrix."""
    r = np.asarray(m, np.float64).copy()
    if from_mitsuba:
        r[:, 0] *= -1
        r[:, 2] *= -1
    else:
        r = r[[2, 0, 1], :]
    r[:, 3] = (r[:, 3] - np.asarray(offset)) / scale
    r[:, 1] *= -1
    r[:, 2] *= -1
    return np.vstack([r, [0, 0, 0, 1]])


def _write_snapshot(path, model, dataset):
    import msgpack

    snapshot.save_snapshot(path, model.desc, model.params, np.zeros(abi.NSB_GRID_CELLS, F32), model.aabb_scale, compress=False)
    cfg = msgpack.unpackb(open(path, "rb").read(), raw=False)
    if dataset is None:
        del cfg["snapshot"]["nerf"]["dataset"]
    else:
        cfg["snapshot"]["nerf"]["dataset"].update(scale=dataset[0], offset=list(dataset[1]), from_mitsuba=False)
    open(path, "wb").write(msgpack.packb(cfg, use_bin_type=True))


def _make_dataset(renderer, model, d, dataset, channels=4, edits=False, n=4):
    """Ground-truth PNGs rendered from the scene for n orbit cameras, and transforms.json with their inverse-mapped matrices."""
    import torch

    cams = syn.orbit_cameras(120)
    base = ev.test_frame(syn.make_frame(model, np.eye(3, 4, dtype=F32), GW, GH))
    frames = []
    os.makedirs(os.path.join(d, "test"), exist_ok=True)
    if edits:
        renderer.set_edit_operators([op.to_op() for op in fx.e1(model)])
        base.apply_operators = 1
    for i in range(n):
        tm = ngp_matrix_to_nerf(cams[10 + 17 * i], *dataset)
        st = ev._camera_state(CAX, tm[:3], dataset)
        _, img = renderer.render_accumulate(ev.sub_frames(base, GW, GH, 8, st), ev._tonemap(False))
        px = renderer.frame_to_rgba8(img, 0.0).cpu().numpy()
        name = f"./test/r_{i}"
        if channels == 4:
            slices.write_png(os.path.join(d, name[2:] + ".png"), px, 4)
        else:
            from PIL import Image

            Image.fromarray(px[..., :3], "RGB").save(os.path.join(d, name[2:] + ".png"))
        frames.append({"file_path": name, "transform_matrix": tm.tolist()})
    if edits:
        renderer.reset_edit_operators()
    torch.cuda.synchronize()
    tj = {"camera_angle_x": CAX, "w": GW, "h": GH, "frames": frames}
    path = os.path.join(d, "transforms_test.json")
    json.dump(tj, open(path, "w"))
    return path


def _transcribed(renderer, model, transforms, dataset, srgb=False, spp=8):
    """run.py's loop with the existing calls (camera_path.render = render_to_cpu) and the restatement with correctly rounded pow."""
    tj = json.load(open(transforms))
    base = ev.test_frame(syn.make_frame(model, np.eye(3, 4, dtype=F32), GW, GH), srgb)
    out = []
    for fj in tj["frames"]:
        px = ev.read_image_u8(ev.find_image(os.path.dirname(transforms), fj["file_path"]))
        ref = er.reference_image(px, srgb and px.shape[2] == 4, (0.0, 0.0, 0.0, 1.0))
        st = ev._camera_state(tj["camera_angle_x"], np.asarray(fj["transform_matrix"])[:-1, :], dataset)
        image = cp.render(renderer, base, None, px.shape[1], px.shape[0], spp, True, state=st, tonemap=ev._tonemap(srgb))
        m = er.metrics(image, ref)
        out.append((float(m["mse"]), float(m["ssim"])))
    return out


@pytest.mark.parametrize("with_dataset", [True, False], ids=["dataset", "no_dataset"])
def test_evaluate_matches_run_py_loop(scene, renderer, tmp_path, with_dataset):
    import torch

    model, _ = scene
    snap = os.path.join(str(tmp_path), "s.msgpack")
    _write_snapshot(snap, model, ((0.45, (0.4, 0.5, 0.55)) if with_dataset else None))
    dataset = snapshot.load_dataset_transform(snap)
    assert (dataset[0] != 1.0) == with_dataset
    tr = _make_dataset(renderer, model, str(tmp_path), dataset)
    base = syn.make_frame(model, np.eye(3, 4, dtype=F32), GW, GH)
    probe_frame = syn.make_frame(model, syn.orbit_cameras(120)[3], GW, GH)
    before, _ = renderer.render(probe_frame)
    before = before.cpu().numpy()
    res = ev.evaluate(renderer, base, tr, dataset=dataset, out_dir=os.path.join(str(tmp_path), "out"))
    want = _transcribed(renderer, model, tr, dataset)
    assert [(m, s) for m, s in zip(res.mse, res.ssim)] == want
    print("evaluate:", res.summary())
    assert res.mean_psnr > 20 and 0.5 < res.mean_ssim <= 1.0
    for f in ("ref.png", "out.png", "diff.png"):
        assert os.path.isfile(os.path.join(str(tmp_path), "out", f))
    res2 = ev.evaluate(renderer, base, tr, dataset=dataset)
    assert res2.mse == res.mse and res2.ssim == res.ssim and res2.summary() == res.summary()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        ev.evaluate(renderer, base, tr, dataset=dataset)
    torch.cuda.synchronize()
    assert torch.cuda.mem_get_info()[0] == free0
    after, _ = renderer.render(probe_frame)
    assert np.array_equal(before, after.cpu().numpy())


def test_evaluate_edited_ground_truth_scores_lower(scene, renderer, tmp_path):
    model, _ = scene
    ds = (1.0, (0.0, 0.0, 0.0), False)
    base = syn.make_frame(model, np.eye(3, 4, dtype=F32), GW, GH)
    plain = ev.evaluate(renderer, base, _make_dataset(renderer, model, os.path.join(str(tmp_path), "a"), ds), dataset=ds)
    edited = ev.evaluate(renderer, base, _make_dataset(renderer, model, os.path.join(str(tmp_path), "b"), ds, edits=True), dataset=ds)
    print("plain:", plain.summary(), "edited:", edited.summary())
    assert edited.mean_psnr < plain.mean_psnr


def test_evaluate_rgb_ground_truth_and_srgb_mode(scene, renderer, tmp_path):
    model, _ = scene
    ds = (1.0, (0.0, 0.0, 0.0), False)
    base = syn.make_frame(model, np.eye(3, 4, dtype=F32), GW, GH)
    for channels in (3, 4):
        tr = _make_dataset(renderer, model, os.path.join(str(tmp_path), f"c{channels}"), ds, channels=channels, n=2)
        for srgb in (False, True):
            res = ev.evaluate(renderer, base, tr, srgb=srgb, dataset=ds)
            assert [(m, s) for m, s in zip(res.mse, res.ssim)] == _transcribed(renderer, model, tr, ds, srgb=srgb), (channels, srgb)
            assert np.isfinite(res.mean_psnr) and np.isfinite(res.mean_ssim)


def test_screenshots(scene, renderer, tmp_path):
    model, _ = scene
    ds = (0.45, (0.4, 0.5, 0.55), False)
    tr = _make_dataset(renderer, model, os.path.join(str(tmp_path), "d"), ds, n=3)
    tj = json.load(open(tr))
    tj["frames"][1]["file_path"] = "./test/r_1.png"
    json.dump(tj, open(tr, "w"))
    base = syn.make_frame(model, np.eye(3, 4, dtype=F32), GW, GH)
    out = os.path.join(str(tmp_path), "shots")
    names = ev.screenshots(renderer, base, tr, out, frames=["0", "1"], spp=4, width=40, height=30, dataset=ds)
    assert names == [os.path.join(out, "r_0.png"), os.path.join(out, "r_1.png")]
    for name, fj in zip(names, tj["frames"][:2]):
        st = ev._camera_state(CAX, np.asarray(fj["transform_matrix"])[:-1, :], ds)
        frame = cp.render(renderer, base, None, 40, 30, 4, True, state=st)
        got = decode_png(open(name, "rb").read())
        _check_bytes(got.reshape(30, 40, 4), frame, 0.0)
    tj["frames"][2]["file_path"] = "./test/r_2.jpg"
    json.dump(tj, open(tr, "w"))
    with pytest.raises(ValueError):
        ev.screenshots(renderer, base, tr, out, frames=["2"], dataset=ds)


def test_cli_prints_run_py_summary(scene, renderer, tmp_path):
    """tools/evaluate.py on a snapshot and a transforms file prints run.py's line, the one evaluate computes for the same context."""
    import sys

    from nerfshop_b200.renderer import NerfRenderer

    model, _ = scene
    d = str(tmp_path)
    snap = os.path.join(d, "s.msgpack")
    _write_snapshot(snap, model, (0.45, (0.4, 0.5, 0.55)))
    ds = snapshot.load_dataset_transform(snap)
    tr = _make_dataset(renderer, model, d, ds, n=2)
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    res = subprocess.run([sys.executable, os.path.join(root, "tools", "evaluate.py"), "--snapshot", snap, "--test_transforms", tr,
                          "--screenshot_transforms", tr, "--screenshot_dir", os.path.join(d, "shots"), "--width", "32", "--height", "24"],
                         capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    line = [ln for ln in res.stdout.splitlines() if ln.startswith("PSNR=")]
    r = NerfRenderer(0)
    desc, params, grid, aabb_scale = snapshot.load_snapshot(snap)
    r.upload_model(desc, params)
    r.upload_density_grid(grid)
    want = ev.evaluate(r, syn.make_frame(model, np.eye(3, 4, dtype=F32), 64, 64), tr, dataset=ds)
    r.close()
    print(line)
    assert line == [want.summary()]
    assert sorted(os.listdir(os.path.join(d, "shots"))) == ["r_0.png", "r_1.png"]
