"""Host restatement of the image-quality metrics (nerfshop_b200/csrc/nsb_eval.cuh): scripts/common.py's read_image, linear_to_srgb,
compute_error("MSE" / "SSIM") and run.py's sRGB blend, in numpy float32 in numpy's operation order, with the pow pluggable.

  pow_cr   correctly rounded float32 pow: float64 pow rounded once, and where that double lies within 2^-40 (relative) of a float32
           rounding boundary, the exact power settled with `decimal` at 60 digits (so the host's float64 pow cannot decide a tie)
  pow_np   numpy's own float32 `**`, whose result depends on the host (SIMD code on AVX-512, libm elsewhere)

Every other step names the numpy operation it restates; tests/test_evaluate_cpu.py checks each against numpy and scipy themselves.
"""
from __future__ import annotations

import decimal

import numpy as np

F32, F64 = np.float32, np.float64
K = np.array([0.120078, 0.233881, 0.292082, 0.233881, 0.120078])  # common.py's SSIM blur kernel
GAMMA = F32(0.4545454545)
C1, C2 = F32(0.01 ** 2), F32(0.03 ** 2)


def _exact_pow(x: float, y: float) -> decimal.Decimal:
    with decimal.localcontext() as ctx:
        ctx.prec = 60
        return decimal.Decimal(x) ** decimal.Decimal(y)


def pow_cr(x, y) -> np.ndarray:
    x = np.asarray(x, F32)
    y = F32(y)
    with np.errstate(all="ignore"):
        d = np.power(x.astype(F64), F64(y))
        r = d.astype(F32)
        # the float32 neighbour on the other side of d and the boundary between them
        other = np.where(d >= r.astype(F64), np.nextafter(r, F32(np.inf)), np.nextafter(r, F32(-np.inf)))
        mid = (r.astype(F64) + other.astype(F64)) / 2
        near = np.isfinite(d) & (d > 0) & (np.abs(d - mid) <= np.abs(d) * 2.0 ** -40)
    if near.any():
        r = r.copy()
        for idx in zip(*np.nonzero(near)) if r.ndim else [()]:
            e = _exact_pow(float(x[idx]), float(y))
            lo, hi = sorted((float(r[idx]), float(other[idx])))
            m = (decimal.Decimal(lo) + decimal.Decimal(hi)) / 2
            if e < m:
                r[idx] = F32(lo)
            elif e > m:
                r[idx] = F32(hi)
            else:  # an exact tie: round half to even
                r[idx] = F32(lo) if (np.array(lo, F32).view(np.uint32) & 1) == 0 else F32(hi)
    return r


def pow_np(x, y) -> np.ndarray:
    with np.errstate(all="ignore"):
        return np.asarray(x, F32) ** F32(y)


# ---- common.py:139-145 ---------------------------------------------------------------------------------------------------
def srgb_to_linear(x, pw=pow_cr) -> np.ndarray:
    x = np.asarray(x, F32)
    with np.errstate(all="ignore"):
        return np.where(x > F32(0.04045), pw((x + F32(0.055)) / F32(1.055), F32(2.4)), x / F32(12.92)).astype(F32)


def linear_to_srgb(x, pw=pow_cr) -> np.ndarray:
    x = np.asarray(x, F32)
    with np.errstate(all="ignore"):
        return np.where(x > F32(0.0031308), F32(1.055) * pw(x, F32(1.0 / 2.4)) - F32(0.055), F32(12.92) * x).astype(F32)


# ---- read_image (common.py:147-161) on 8-bit pixels, and run.py's sRGB blend (run.py:264-270) --------------------------------
def reference_image(px, srgb_blend: bool = False, background=(0.0, 0.0, 0.0, 1.0), pw=pow_cr) -> np.ndarray:
    """uint8 [H, W, 3 or 4] -> float32 [H, W, 4], linear premultiplied; RGB gets alpha 1."""
    img = np.asarray(px).astype(F32) / F32(255.0)
    if img.shape[2] == 3:
        out = np.ones(img.shape[:2] + (4,), F32)
        out[..., :3] = srgb_to_linear(img, pw)
        return out
    img[..., 0:3] = srgb_to_linear(img[..., 0:3], pw)
    img[..., 0:3] *= img[..., 3:4]
    if srgb_blend:
        with np.errstate(all="ignore"):
            img[..., :3] = np.divide(img[..., :3], img[..., 3:4], out=np.zeros_like(img[..., :3]), where=img[..., 3:4] != 0)
        img[..., :3] = linear_to_srgb(img[..., :3], pw)
        img[..., :3] *= img[..., 3:4]
        img += (F32(1.0) - img[..., 3:4]) * np.asarray(background, F32)
        img[..., :3] = srgb_to_linear(img[..., :3], pw)
    return img


# ---- run.py:286-290 ----------------------------------------------------------------------------------------------------
def clip01(x) -> np.ndarray:
    return np.clip(np.asarray(x, F32), F32(0.0), F32(1.0))


def metric_r(rgb, pw=pow_cr) -> np.ndarray:
    """R = np.clip(linear_to_srgb(ref[..., :3]), 0, 1)."""
    return clip01(linear_to_srgb(rgb, pw))


def metric_a(rgb, pw=pow_cr) -> np.ndarray:
    """A, then compute_error_img's clean-up: non-finite -> 0, np.maximum(., 0)."""
    a = metric_r(rgb, pw)
    a[np.logical_not(np.isfinite(a))] = 0
    return np.maximum(a, F32(0.0))


def luminance(c, pw=pow_cr) -> np.ndarray:
    """common.py:186-188 on np.clip(c, 0, 1)."""
    p = pw(np.maximum(F32(0.0), clip01(c)), GAMMA)
    return F32(0.2126) * p[..., 0] + F32(0.7152) * p[..., 1] + F32(0.0722) * p[..., 2]


def mse_map(A, R) -> np.ndarray:
    """compute_error("MSE")'s map: L2, non-finite -> 0, the channel mean as float32(float64((s0 + s1) + s2) / 3)."""
    with np.errstate(all="ignore"):
        s = (A - R) ** 2
    s[np.logical_not(np.isfinite(s))] = 0
    return ((s[..., 0] + s[..., 1] + s[..., 2]).astype(F64) / 3).astype(F32)


def blur_axis(x, axis: int) -> np.ndarray:
    """convolve1d(x, K, axis, mode='reflect') on float32: the symmetric-kernel loop in float64, x0 * k2 + (x-2 + x2) * k0 + (x-1 + x1) * k1,
    rounded once to float32."""
    x = np.moveaxis(np.asarray(x, F32), axis, 0).astype(F64)
    n = x.shape[0]
    idx = np.arange(-2, n + 2)
    while ((idx < 0) | (idx >= n)).any():
        idx = np.where(idx < 0, -idx - 1, np.where(idx >= n, 2 * n - 1 - idx, idx))
    p = x[idx]
    t = p[2:n + 2] * K[2]
    t = t + (p[0:n] + p[4:n + 4]) * K[0]
    t = t + (p[1:n + 1] + p[3:n + 3]) * K[1]
    return np.moveaxis(t.astype(F32), 0, axis)


def blur(x) -> np.ndarray:
    return blur_axis(blur_axis(x, 0), 1)


def ssim_map(la, lb) -> np.ndarray:
    """SSIM (common.py:190-207) after the luminance, then compute_error's non-finite -> 0."""
    with np.errstate(all="ignore"):
        mA, mB = blur(la), blur(lb)
        sA = blur(la * la) - mA * mA
        sB = blur(lb * lb) - mB * mB
        sAB = blur(la * lb) - mA * mB
        p1 = (F32(2.0) * mA * mB + C1) / (mA * mA + mB * mB + C1)
        p2 = (F32(2.0) * sAB + C2) / (sA + sB + C2)
        e = p1 * p2
    e[np.logical_not(np.isfinite(e))] = 0
    return e


# ---- np.mean of a map: numpy's pairwise float32 sum ----------------------------------------------------------------------------
def _split(n: int) -> int:
    h = n // 2
    return h - h % 8


def _leaves(off: int, n: int, out: list) -> None:
    if n <= 128:
        out.append((off, n))
        return
    n2 = _split(n)
    _leaves(off, n2, out)
    _leaves(off + n2, n - n2, out)


def _leaf_sum(a, n: int) -> np.ndarray:
    """numpy's leaf for rows a[:, :n] of equal length n: n < 8 in order from -0.0, else eight strided accumulators and the tail."""
    if n < 8:
        r = np.full(a.shape[0], -0.0, F32)
        for i in range(n):
            r = r + a[:, i]
        return r
    m = n - n % 8
    r = a[:, 0:8].copy()
    for i in range(8, m, 8):
        r = r + a[:, i:i + 8]
    res = ((r[:, 0] + r[:, 1]) + (r[:, 2] + r[:, 3])) + ((r[:, 4] + r[:, 5]) + (r[:, 6] + r[:, 7]))
    for i in range(m, n):
        res = res + a[:, i]
    return res


def pairwise_sum(flat) -> np.float32:
    """numpy's pairwise_sum of a contiguous float32 array (loops_utils.h.src)."""
    a = np.ascontiguousarray(flat, F32).reshape(-1)
    leaves = []
    _leaves(0, a.size, leaves)
    sums = {}
    for n in sorted({n for _, n in leaves}):
        offs = np.array([o for o, m in leaves if m == n], np.int64)
        rows = a[offs[:, None] + np.arange(n)[None, :]]
        for o, s in zip(offs.tolist(), _leaf_sum(rows, n)):
            sums[o] = F32(s)

    def rec(off, n):
        if n <= 128:
            return sums[off]
        n2 = _split(n)
        return F32(rec(off, n2) + rec(off + n2, n - n2))

    with np.errstate(all="ignore"):
        return rec(0, a.size)


def np_mean(m) -> np.float32:
    """np.mean of a C-contiguous float32 map: float32(float64(pairwise_sum) / n)."""
    return F32(F64(pairwise_sum(m)) / np.asarray(m).size)


def metrics(image, ref, pw=pow_cr) -> dict:
    """run.py's per-frame block on float32 [H, W, 4] frames: A, R, both luminances, both maps and both means."""
    A = metric_a(np.asarray(image, F32)[..., :3], pw)
    R = metric_r(np.asarray(ref, F32)[..., :3], pw)
    la, lb = luminance(A, pw), luminance(R, pw)
    mm, sm = mse_map(A, R), ssim_map(la, lb)
    return {"A": A, "R": R, "la": la, "lb": lb, "mse_map": mm, "ssim_map": sm, "mse": np_mean(mm), "ssim": np_mean(sm)}


def ulps(a, b) -> np.ndarray:
    """|a - b| in float32 ulps (same-sign finite values)."""
    ia = np.asarray(a, F32).view(np.int32).astype(np.int64)
    ib = np.asarray(b, F32).view(np.int32).astype(np.int64)
    return np.abs(ia - ib)
