"""The image-quality metrics without a GPU: the host restatement (tests/eval_rule.py) against numpy and scipy themselves and against the
reference's own scripts/common.py, the float32 camera of nerf_matrix_to_ngp, run.py's file lookup, the snapshot's dataset transform and
the ground-truth decoder's errors.

The reference's common.py is imported where its sources exist (NSB_REFERENCE_ROOT), with stand-ins for the modules it imports but does not
use here (imageio, backed by PIL, and flip); its results are stored under tests/golden/ref/test_evaluate_cpu/ with NSB_RECORD_REF_GOLDEN=1
and replayed elsewhere: the stages after the pows exactly, the stages through a pow within a few ulps (numpy's float32 pow depends on the
host and is 1 ulp off the correctly rounded one on about a fifth of inputs on AVX-512)."""
import importlib.util
import os
import sys
import types

import msgpack
import numpy as np
import pytest
from scipy.ndimage import convolve1d

import eval_rule as er
from nerfshop_b200 import evaluate as ev
from nerfshop_b200 import slices, snapshot
from nerfshop_b200 import synthetic as syn

F32 = np.float32
REF = os.environ.get("NSB_REFERENCE_ROOT", "/root/reference")
COMMON = os.path.join(REF, "scripts", "common.py")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref", "test_evaluate_cpu", "common_py.npz")
RECORD = os.environ.get("NSB_RECORD_REF_GOLDEN") == "1"
CRAFTED = np.array([1e30, -1e30, 1.0, 1e-30, 1e-45, 3e-39, -2.5, 0.7, 1e8, -1e8, 0.0, -0.0], F32)


def _same(a, b) -> bool:
    return np.array_equal(np.asarray(a, F32).view(np.uint32), np.asarray(b, F32).view(np.uint32))


# ---- the restatement against numpy / scipy ----------------------------------------------------------------------------------
def test_pairwise_mean_every_length_to_4096():
    rng = np.random.default_rng(1)
    for n in range(1, 4097):
        a = (rng.standard_normal(n) * rng.choice(np.array([1e-3, 1.0, 1e3], F32), n)).astype(F32)
        assert _same(er.np_mean(a), np.mean(a)), n


@pytest.mark.parametrize("shape", [(800, 800), (1920, 1080), (1080, 1920), (333, 517), (1, 7), (7, 1)])
def test_pairwise_mean_frame_sizes(shape):
    m = np.random.default_rng(2).random(shape, dtype=F32)
    assert _same(er.np_mean(m), np.mean(m))
    assert _same(er.np_mean(-m), np.mean(-m))


def test_blur_equals_convolve1d():
    rng = np.random.default_rng(3)
    for H in range(1, 8):
        for W in range(1, 8):
            for trial in range(24):
                x = rng.choice(CRAFTED, (H, W)) if trial % 2 else rng.random((H, W), dtype=F32)
                ref = convolve1d(convolve1d(x, er.K, axis=0), er.K, axis=1)
                assert _same(er.blur(x), ref), (H, W, trial)


def test_blur_tap_order_is_pinned():
    """The crafted magnitudes tell convolve1d's order from a left-to-right 5-tap sum: the restatement follows the former."""
    rng = np.random.default_rng(4)
    k = er.K

    def left_to_right(x, axis):
        x = np.moveaxis(x, axis, 0).astype(np.float64)
        n = x.shape[0]
        idx = np.arange(-2, n + 2)
        while ((idx < 0) | (idx >= n)).any():
            idx = np.where(idx < 0, -idx - 1, np.where(idx >= n, 2 * n - 1 - idx, idx))
        p = x[idx]
        t = p[0:n] * k[0] + p[1:n + 1] * k[1] + p[2:n + 2] * k[2] + p[3:n + 3] * k[3] + p[4:n + 4] * k[4]
        return np.moveaxis(t.astype(F32), 0, axis)

    differ = 0
    for _ in range(200):
        x = rng.choice(CRAFTED, (6, 6))
        ref = convolve1d(convolve1d(x, k, axis=0), k, axis=1)
        assert _same(er.blur(x), ref)
        differ += not _same(left_to_right(left_to_right(x, 0), 1), ref)
    assert differ > 0


def test_channel_mean():
    rng = np.random.default_rng(5)
    t = (rng.random((200, 100, 3), dtype=F32) * rng.choice(np.array([1e-3, 1.0, 1e3], F32), (200, 100, 3))).astype(F32)
    s = t ** 2
    assert _same(er.mse_map(t, np.zeros_like(t)), np.mean(s, axis=2))


def _numpy_chain(image, ref):
    """run.py:286-288 + common.py's compute_error, transcribed (numpy's own pow)."""
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
    return A, R, a, b, np.mean(m, axis=2), e, mse, np.mean(e)


def _image_pair(seed, H=37, W=53):
    rng = np.random.default_rng(seed)
    ref = rng.random((H, W, 4), dtype=F32)
    img = np.clip(ref + F32(0.05) * rng.standard_normal((H, W, 4)).astype(F32), -0.2, 1.5).astype(F32)
    img.reshape(-1, 4)[rng.choice(H * W, 12, replace=False), rng.integers(0, 3, 12)] = rng.choice(
        np.array([np.nan, np.inf, -np.inf, 1e4, -1.0, 0.0031308, 0.04045], F32), 12)
    return img, ref


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_restatement_with_numpy_pow_equals_numpy(seed):
    img, ref = _image_pair(seed)
    A, R, a, b, mm, sm, mse, ssim = _numpy_chain(img, ref)
    got = er.metrics(img, ref, er.pow_np)
    for k, want in (("A", A), ("R", R), ("la", a), ("lb", b), ("mse_map", mm), ("ssim_map", sm), ("mse", mse), ("ssim", ssim)):
        assert _same(got[k], want), k


def test_pow_cr_is_correctly_rounded_and_numpy_pow_within_an_ulp():
    x = np.random.default_rng(6).random(200_000, dtype=F32)
    for y in (F32(1.0 / 2.4), F32(2.4), er.GAMMA):
        cr = er.pow_cr(x, y)
        for i in range(0, x.size, 20_000):  # spot checks against the exact power
            e = er._exact_pow(float(x[i]), float(y))
            lo, hi = np.nextafter(cr[i], F32(0)), np.nextafter(cr[i], F32(2))
            assert abs(e - er.decimal.Decimal(float(cr[i]))) <= min(abs(e - er.decimal.Decimal(float(lo))), abs(e - er.decimal.Decimal(float(hi))))
        d = er.ulps(cr, er.pow_np(x, y))
        print(f"pow {float(y):.9g}: numpy's float32 pow differs from the correctly rounded one on {int((d > 0).sum())} of {x.size}, max {int(d.max())} ulp")
        assert d.max() <= 1


# ---- the reference's own common.py --------------------------------------------------------------------------------------------
def _import_common():
    imageio = types.ModuleType("imageio")

    def imread(path):
        from PIL import Image

        with Image.open(path) as im:
            return np.array(im)

    imageio.imread = imread
    flip = types.ModuleType("flip")
    flip.utils = types.ModuleType("flip.utils")
    saved = {k: sys.modules.get(k) for k in ("imageio", "flip", "flip.utils")}
    sys.modules.update({"imageio": imageio, "flip": flip, "flip.utils": flip.utils})
    try:
        spec = importlib.util.spec_from_file_location("nsb_ref_common", COMMON)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return mod
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def _common_results(common, tmp_path):
    """The reference's functions on seeded pairs and on PNG files written with slices.write_png."""
    out = {}
    for seed in (0, 1, 2):
        img, ref = _image_pair(seed)
        A = np.clip(common.linear_to_srgb(img[..., :3]), 0.0, 1.0)
        R = np.clip(common.linear_to_srgb(ref[..., :3]), 0.0, 1.0)
        out[f"img{seed}"], out[f"ref{seed}"] = img, ref
        out[f"A{seed}"], out[f"R{seed}"] = A, R
        out[f"mse{seed}"] = np.float32(common.compute_error("MSE", A.copy(), R))
        out[f"ssim{seed}"] = np.float32(common.compute_error("SSIM", A.copy(), R))
        A0 = A.copy()
        A0[np.logical_not(np.isfinite(A0))] = 0
        A0 = np.maximum(A0, 0.0)
        out[f"la{seed}"], out[f"lb{seed}"] = common.luminance(A0), common.luminance(R)
        out[f"ssim_map{seed}"] = common.SSIM(A0, R)
        out[f"psnr{seed}"] = np.float64(common.mse2psnr(float(out[f"mse{seed}"])))
    rng = np.random.default_rng(7)
    px = rng.integers(0, 256, (16, 16, 4), dtype=np.uint8)
    px[0, :, 3] = 0
    name = os.path.join(str(tmp_path), "gt.png")
    slices.write_png(name, px, 4)
    out["png_px"] = px
    out["png_read"] = common.read_image(name)
    return out


@pytest.fixture(scope="module")
def common_results(tmp_path_factory):
    if os.path.isfile(COMMON):
        res = _common_results(_import_common(), tmp_path_factory.mktemp("common"))
        if RECORD:
            os.makedirs(os.path.dirname(GOLDEN), exist_ok=True)
            np.savez_compressed(GOLDEN, **res)
        return res, True
    if not os.path.isfile(GOLDEN):
        pytest.skip("neither the reference's scripts/common.py nor its stored results")
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}, False


def test_restatement_equals_reference_common(common_results):
    res, live = common_results
    for seed in (0, 1, 2):
        img, ref = res[f"img{seed}"], res[f"ref{seed}"]
        if live:  # the same host: with numpy's pow, bit for bit at every stage
            got = er.metrics(img, ref, er.pow_np)
            for k in ("R", "la", "lb", "ssim_map", "mse", "ssim"):
                assert _same(got[k], res[f"{k}{seed}"]), (seed, k)
            assert ev.mse2psnr(float(got["mse"])) == float(res[f"psnr{seed}"])
        # the stages after the pows, fed the reference's own A, R and luminances: exact on every host
        A0 = er.metric_a(img[..., :3], er.pow_np) if live else None
        R = res[f"R{seed}"]
        la, lb = res[f"la{seed}"], res[f"lb{seed}"]
        assert _same(er.ssim_map(la, lb), res[f"ssim_map{seed}"])
        assert _same(er.np_mean(res[f"ssim_map{seed}"]), res[f"ssim{seed}"])
        A = res[f"A{seed}"].copy()
        A[np.logical_not(np.isfinite(A))] = 0
        A = np.maximum(A, F32(0))
        assert _same(er.np_mean(er.mse_map(A, R)), res[f"mse{seed}"])
        if A0 is not None:
            assert _same(A0, A)
        # the pow stages, correctly rounded: a pow that is 1 ulp off numpy's moves R by a few ulps where 1.055 * p - 0.055 cancels
        got = er.metrics(img, ref, er.pow_cr)
        for k in ("R", "la", "lb"):
            assert er.ulps(got[k], res[f"{k}{seed}"]).max() <= 8, (seed, k)
    px = res["png_px"]
    want = res["png_read"]
    got_np = er.reference_image(px, pw=er.pow_np)
    if live:
        assert _same(got_np, want)
    assert er.ulps(er.reference_image(px), want).max() <= 2  # the pow, then the product with alpha


# ---- the camera -------------------------------------------------------------------------------------------------------
def test_nerf_matrix_to_ngp_default_dataset_matches_synthetic_float64_version_closely():
    m = syn.FOX_FRAME0
    a = ev.nerf_matrix_to_ngp(m, 0.33, (0.5, 0.5, 0.5))
    b = syn.nerf_matrix_to_ngp(m)
    assert a.dtype == F32 and np.abs(a - b).max() <= 1e-6


@pytest.mark.parametrize("from_mitsuba", [False, True])
def test_nerf_matrix_to_ngp_float32_steps(from_mitsuba):
    rng = np.random.default_rng(8)
    m = rng.standard_normal((3, 4)) * 3
    scale, offset = 0.7123, (0.25, -1.5, 3.0)
    r = np.array(m, F32)
    r[:, 1:3] *= -1
    col = r[:, 3] * F32(scale)
    r[:, 3] = col + np.array(offset, F32)
    want = r * np.array([-1, 1, -1, 1], F32) if from_mitsuba else r[[1, 2, 0]]
    assert _same(ev.nerf_matrix_to_ngp(m, scale, offset, from_mitsuba), want)
    assert _same(ev.nerf_matrix_to_ngp(m), np.array(m, F32)[[1, 2, 0]] * np.array([1, -1, -1, 1], F32))


# ---- parsing and lookup ----------------------------------------------------------------------------------------------
def test_find_image_follows_run_py(tmp_path):
    d = str(tmp_path)
    os.makedirs(os.path.join(d, "test"))
    px = np.zeros((2, 2, 4), np.uint8)
    slices.write_png(os.path.join(d, "test", "r_0.png"), px, 4)
    assert ev.find_image(d, "./test/r_0") == os.path.join(d, "./test/r_0.png")  # has a '.', so .png is appended by the second try
    assert ev.find_image(d, "test/r_0") == os.path.join(d, "test/r_0.png")      # no '.': .png appended first
    open(os.path.join(d, "test", "r_1.jpg"), "wb").close()
    assert ev.find_image(d, "./test/r_1") == os.path.join(d, "./test/r_1.jpg")
    assert ev.find_image(d, "test/r_9") == os.path.join(d, "test/r_9.png.exr")


def test_read_image_errors(tmp_path):
    from PIL import Image

    d = str(tmp_path)
    Image.fromarray(np.zeros((4, 4), np.uint8), "L").save(os.path.join(d, "grey.png"))
    Image.fromarray(np.zeros((4, 4), np.uint16)).save(os.path.join(d, "deep.png"))
    for name in ("grey.png", "deep.png", "x.exr"):
        with pytest.raises(ValueError):
            ev.read_image_u8(os.path.join(d, name))
    with pytest.raises(FileNotFoundError):
        ev.read_image_u8(os.path.join(d, "missing.png"))
    px = np.random.default_rng(9).integers(0, 256, (5, 3, 4), dtype=np.uint8)
    slices.write_png(os.path.join(d, "ok.png"), px, 4)
    assert np.array_equal(ev.read_image_u8(os.path.join(d, "ok.png")), px)


def test_snapshot_dataset_transform(tmp_path):
    model = syn.make_model(seed=1337)
    p = os.path.join(str(tmp_path), "s.msgpack")
    snapshot.save_snapshot(p, model.desc, model.params, np.zeros(5 * 128 ** 3, F32), 16, compress=False)
    assert snapshot.load_dataset_transform(p) == (pytest.approx(0.33), (0.5, 0.5, 0.5), False)
    cfg = msgpack.unpackb(open(p, "rb").read(), raw=False)
    cfg["snapshot"]["nerf"]["dataset"].update(scale=0.8, offset=[0.1, 0.2, 0.3], from_mitsuba=True)
    open(p, "wb").write(msgpack.packb(cfg, use_bin_type=True))
    assert snapshot.load_dataset_transform(p) == (pytest.approx(0.8), (pytest.approx(0.1), pytest.approx(0.2), pytest.approx(0.3)), True)
    del cfg["snapshot"]["nerf"]["dataset"]  # export_snapshot's form
    open(p, "wb").write(msgpack.packb(cfg, use_bin_type=True))
    assert snapshot.load_dataset_transform(p) == (1.0, (0.0, 0.0, 0.0), False)
    assert snapshot.load_snapshot(p)[3] == 16
