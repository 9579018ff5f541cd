"""Inputs of the frame post-process (accumulate_kernel / tonemap_kernel and nsb_accumulate / nsb_tonemap) over their whole domain: the
case tables of test_gpu_postprocess_domain.py.

Pixels come in classes. The finite ones are compared bit for bit; NON_FINITE (and the -0 entries of TINY) also reach the places where
the reference's Eigen stand-in (a < b ? b : a) and real Eigen on the device (fmaxf / fminf) part ways, see the rule in the GPU test.
"""
import numpy as np

from nerfshop_b200 import abi

F32 = np.float32
SRGB_LINEAR_EDGE = F32(0.0031308)  # linear_to_srgb's branch
SRGB_EDGE = F32(0.04045)           # srgb_to_linear's branch


def _ulps(x, k=2):
    """x and its k float32 neighbours on each side."""
    out, lo, hi = [F32(x)], F32(x), F32(x)
    for _ in range(k):
        lo, hi = np.nextafter(lo, F32(-np.inf)), np.nextafter(hi, F32(np.inf))
        out += [lo, hi]
    return np.array(out, F32)


def _alpha(rng, n, lo=0.0, hi=1.0):
    return rng.uniform(lo, hi, n).astype(F32)


def pixels(cls: str, n: int, seed: int = 0) -> np.ndarray:
    """n RGBA pixels [n, 4] of input class `cls`."""
    rng = np.random.default_rng(seed + 7919 * CLASSES.index(cls))
    if cls == "unit":          # premultiplied values in [0, 1]
        p = rng.random((n, 4), dtype=F32)
        p[:, :3] *= p[:, 3:4]
    elif cls == "hdr":         # up to 1e4, log-uniform from 1e-3
        p = np.empty((n, 4), F32)
        p[:, :3] = 10.0 ** rng.uniform(-3.0, 4.0, (n, 3))
        p[:, 3] = _alpha(rng, n)
    elif cls == "negative":    # negative colours, alpha outside [0, 1]
        p = rng.uniform(-2.0, 1.0, (n, 4)).astype(F32)
        p[:, 3] = _alpha(rng, n, -0.5, 1.5)
    elif cls == "srgb_edges":  # both branch points of the sRGB curves and their ulp neighbours, in every channel
        v = np.concatenate([_ulps(SRGB_LINEAR_EDGE), _ulps(SRGB_EDGE)])
        p = v[rng.integers(0, v.size, (n, 4))]
        p[:, 3] = np.where(rng.random(n) < 0.5, p[:, 3], _alpha(rng, n))
    elif cls == "tiny":        # subnormals and signed zeros
        v = np.array([0.0, -0.0, 1e-45, -1e-45, 1e-40, -1e-40, 1.1754942e-38, -1.1754942e-38, 1.17549435e-38], F32)
        p = v[rng.integers(0, v.size, (n, 4))]
        p[: n // 2, 3] = _alpha(rng, n // 2)
    elif cls == "nonfinite":   # +-inf and NaN in any channel, next to ordinary values
        p = rng.random((n, 4), dtype=F32)
        v = np.array([np.inf, -np.inf, np.nan], F32)
        hit = rng.random((n, 4)) < 0.4
        p[hit] = v[rng.integers(0, 3, int(hit.sum()))]
    else:
        raise KeyError(cls)
    return np.ascontiguousarray(p, F32)


CLASSES = ["unit", "hdr", "negative", "srgb_edges", "tiny", "nonfinite"]
FINITE_CLASSES = CLASSES[:-1]

SHAPES = {"1x1": (1, 1), "1xW": (1, 301), "Hx1": (257, 1), "37x53": (37, 53), "1920x1080": (1080, 1920)}  # (H, W)
COLOR_SPACES = {"linear": abi.NSB_COLOR_LINEAR, "srgb": abi.NSB_COLOR_SRGB, "visposneg": abi.NSB_COLOR_VISPOSNEG}
CURVES = {"identity": abi.NSB_TONEMAP_IDENTITY, "aces": abi.NSB_TONEMAP_ACES, "hable": abi.NSB_TONEMAP_HABLE, "reinhard": abi.NSB_TONEMAP_REINHARD}
SEQUENCE = 33                                      # continued accumulations: every prefix (1, 8, ..., 33 calls) is compared
STARTS = (0, 1, 255, 2**24 - 1, 2**24, 2**24 + 1)  # (float)spp + 1 starts to round at 2^24
BIG_STARTS, BIG_SEQUENCE = (0, 2**24), 8           # 1920x1080: fewer, shorter sequences
EXPOSURES = (0.0, 0.5, -0.5, 1.3, -1.3, 20.0, -20.0)
_e = _ulps(SRGB_EDGE, 1)
BACKGROUNDS = (
    (0.0, 0.0, 0.0, 1.0),
    (0.1, 0.2, 0.3, 0.5),
    (0.3, 0.6, 0.9, 0.0),                                  # alpha 0
    (float(_e[1]), float(_e[0]), float(_e[2]), 1.0),       # 0.04045 and its ulp neighbours
    (1.5, 2.0, 7.0, 0.75),                                 # components above 1
)


def frame(shape, seed: int, classes=CLASSES) -> np.ndarray:
    """An [H, W, 4] frame whose pixels are drawn from `classes`, equally often, in a seeded shuffle."""
    H, W = shape
    n = H * W
    per = -(-n // len(classes))
    p = np.concatenate([pixels(c, per, seed) for c in classes])
    rng = np.random.default_rng(seed)
    return np.ascontiguousarray(p[rng.permutation(p.shape[0])[:n]].reshape(H, W, 4))


def tonemap_input(seed: int = 0) -> np.ndarray:
    """The crafted accumulation tonemapped under every parameter set: 40 pixels of each class, [16, 15, 4]."""
    return np.ascontiguousarray(np.concatenate([pixels(c, 40, seed) for c in CLASSES]).reshape(16, 15, 4))


def tonemap_params(cs: int, curve: int, exposures=EXPOSURES, backgrounds=BACKGROUNDS):
    """NsbTonemaps over output space x clamp x exposure x background for one input colour space and curve."""
    out = []
    for out_cs in (abi.NSB_COLOR_LINEAR, abi.NSB_COLOR_SRGB):
        for clamp in (0, 1):
            for e in exposures:
                for bg in backgrounds:
                    p = abi.NsbTonemap()
                    p.color_space, p.output_color_space, p.tonemap_curve, p.clamp_output_color, p.exposure = cs, out_cs, curve, clamp, e
                    p.background_color[:] = bg
                    out.append(p)
    return out


def special(x: np.ndarray) -> np.ndarray:
    """Per pixel of x [..., 4]: a NaN, an inf or a -0 in any channel."""
    return (~np.isfinite(x) | ((x == 0) & np.signbit(x))).any(-1)
