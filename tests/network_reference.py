"""A float64 reference of the fully fused network (hash-grid features -> density MLP -> SH -> rgb MLP), in numpy, and the models that
pin the device's wgmma MLPs against it.

Exact models ("integer" models). The encoding is n_levels 16, F 2, base_resolution 17, per_level_scale 1.0: every level has scale 16
and is a dense 17^3 grid (4,920 entries). At x = (k - 0.5)/16, fma(16, x, 0.5) = k exactly, so the interpolation weight is 0 and
the features are table entries. Tables and weights are small integers times powers of two. `certificate` proves, for every row, layer
and output, that every term is a multiple of the layer's unit u and that sum |w x| <= min(2048 u, 65504): every partial sum in any
order is then an exact fp16 value, so both accumulator policies and any internal precision or rounding of the MMA must give the
float64 result bit for bit. W5 row 3 is the one weight row no output shows (nsb_inference row 3 is the density), so coverage leaves it
out.

SH probes. W3 has one non-zero per row, in an SH column; W4 is a permutation and W5 adds the +/- pair of each column back, all with
power-of-two scales: the rgb outputs are the fp16 SH values of the direction, from `sh4_f32`, a float32 restatement of encode_sh4
in the device's non-contracted mul / sub / add order.

Range models. Integer models scaled by powers of two: subnormal hidden values and outputs down to 2^-24; outputs past 2^14; one
L1 unit pushed past 65504 (-> inf) on the rows whose feature is >= 2, whose successors then see 0 * inf = NaN in every output,
through zero weights too, and ReLU maps NaN to 0 (tcnn's `x > 0 ? x : 0`, the oracle's `!(a > 0)`, the device's __hmax2). Rows
with NaN or +-inf positions have NaN features, so all of L1 is NaN, ReLU gives 0, the density outputs are 0 and rgb is the network
on a zero density input.

Interval forward (random models). Every fp16 activation is an interval [lo, hi] of fp16 values, propagated in float64; each layer
output is rounded outward to fp16, so either fp16 neighbour of any value inside is allowed. The MMA's internal error is bounded at
fp32 level, never looser:
  fp32 accumulators:  products exact, |sum - exact| <= K * 2^-23 * sum |w x| (K = the layer's width), then one fp16 rounding;
  fp16 accumulators:  after every K=16 instruction one fp16 rounding of (acc + the 16 products) with an internal error of at most
                      EPS16 = 17 * 2^-23 times (|acc| + sum of the 16 |w x|).
The rounding is characterised on the device by test_gpu_network_domain.py::test_accumulator_rounding_characterised, with designed
sub-ulp fractions inside one K-chunk: on an H100, m64nNk16 with an fp16 D rounds to nearest, ties to even, once per instruction, and
keeps 2049 + 2^-14 apart from the tie 2049 (more than fp32's 24 bits inside one instruction), so its internal error is below 2^-26
relative there; fp32 accumulators hold 24 bits and __floats2half2_rn rounds to nearest even. Both EPS bounds are fp32 level, looser than
the hardware, and the outward rounding to either fp16 neighbour covers both rounding directions.
Widths (`width_ulps`: hi - lo in fp16 ulps of the output row's largest magnitude), measured over 40,000 `random_rows` of each model:
                        density outputs (max over rows, per policy)   rgb outputs (max)
  fox                   fp32 7,  fp16 14                              fp32 127, fp16 287
  seed 7, gain 1.6      fp32 5,  fp16 11                              fp32 337, fp16 621
  seed 8, gain 2        fp32 5,  fp16 9                               fp32 263, fp16 468
The rgb intervals widen through three layers (plain interval arithmetic keeps no correlation between units), so they catch gross
errors; the exact models are what pins the rgb MLP to the bit. WIDTH_CAP bounds both so the check keeps its teeth.
"""
from __future__ import annotations

import numpy as np

from nerfshop_b200 import abi

SHAPES = [(64, 32), (16, 64), (64, 32), (64, 64), (16, 64)]  # W1 .. W5, [out x in], row-major in the parameter block
N_MLP = sum(o * i for o, i in SHAPES)
N_LEVELS, RES, ENTRIES = 16, 17, 4920
DESC_ARGS = (16, 2, 19, 17, 1.0, 64, 1, 2, 4)
EPS32 = 2.0 ** -23
EPS16 = 17 * 2.0 ** -23
WIDTH_CAP = (16, 1024)  # fp16 ulps of the output's scale (width_ulps): density outputs, rgb outputs


def desc() -> abi.NsbModelDesc:
    return abi.NsbModelDesc(*DESC_ARGS)


# ---- parameter blocks ------------------------------------------------------------------------------------------------
def pack(ws, table) -> np.ndarray:
    """fp16 parameter block [W1 .. W5 | grid] as uint16; table: [16, 4920, 2]."""
    parts = [np.asarray(w, np.float64).reshape(-1) for w in ws] + [np.asarray(table, np.float64).reshape(-1)]
    v = np.concatenate(parts)
    h = v.astype(np.float16)
    assert np.array_equal(h.astype(np.float64), v), "model values must be fp16 values"
    return h.view(np.uint16)


def unpack(params: np.ndarray):
    h = np.asarray(params, np.uint16).view(np.float16).astype(np.float64)
    ws, off = [], 0
    for o, i in SHAPES:
        ws.append(h[off:off + o * i].reshape(o, i))
        off += o * i
    return ws, h[off:]


# ---- positions and features of the exact models ---------------------------------------------------------------------
def lattice_x(k) -> np.ndarray:
    """The float32 position whose fma(16, x, 0.5) is the integer k."""
    x = ((np.asarray(k, np.float64) - 0.5) / 16.0).astype(np.float32)
    assert np.array_equal(np.float64(16.0) * x.astype(np.float64) + 0.5, np.asarray(k, np.float64))
    return x


def lattice_coords(kxyz: np.ndarray, dirs: np.ndarray) -> np.ndarray:
    """NerfCoordinate rows at integer lattice coordinates kxyz [n, 3] with warped directions dirs [n, 3]."""
    c = np.zeros((kxyz.shape[0], 7), np.float32)
    c[:, :3] = lattice_x(kxyz)
    c[:, 3] = 0.01
    c[:, 4:] = dirs
    return c


def table_features(table: np.ndarray, kxyz: np.ndarray) -> np.ndarray:
    """[n, 32] float64: the dense lower-corner entry of every level, the index in tcnn's uint32 arithmetic modulo the level size."""
    g = np.asarray(kxyz, np.int64).astype(np.uint64) & np.uint64(0xFFFFFFFF)
    idx = (g[:, 0] + g[:, 1] * np.uint64(RES) + g[:, 2] * np.uint64(RES * RES)) & np.uint64(0xFFFFFFFF)
    idx = (idx % np.uint64(ENTRIES)).astype(np.int64)
    t = np.asarray(table, np.float64).reshape(N_LEVELS, ENTRIES, 2)
    return t[:, idx, :].transpose(1, 0, 2).reshape(-1, 2 * N_LEVELS)


# ---- SH ------------------------------------------------------------------------------------------------------------
_F = np.float32


def sh4_f32(dw: np.ndarray) -> np.ndarray:
    """[n, 16] float64 of fp16 values: encode_sh4 (nsb_device.cuh) in float32, one rounding per mul / sub / add."""
    dw = np.asarray(dw, np.float32)
    with np.errstate(all="ignore"):
        x, y, z = [(dw[:, a].astype(np.float64) * 2.0 - 1.0).astype(np.float32) for a in range(3)]  # fma(d, 2, -1): d * 2 is exact
        xy, xz, yz, x2, y2, z2 = x * y, x * z, y * z, x * x, y * y, z * z
        o = [np.full_like(x, _F(0.28209479177387814)),
             _F(-0.48860251190291987) * y, _F(0.48860251190291987) * z, _F(-0.48860251190291987) * x,
             _F(1.0925484305920792) * xy, _F(-1.0925484305920792) * yz,
             _F(0.94617469575755997) * z2 - _F(0.31539156525251999),
             _F(-1.0925484305920792) * xz,
             _F(0.54627421529603959) * x2 - _F(0.54627421529603959) * y2,
             (_F(0.59004358992664352) * y) * (_F(-3.0) * x2 + y2),
             (_F(2.8906114426405538) * xy) * z,
             (_F(0.45704579946446572) * y) * (_F(1.0) - _F(5.0) * z2),
             (_F(0.3731763325901154) * z) * (_F(5.0) * z2 - _F(3.0)),
             (_F(0.45704579946446572) * x) * (_F(1.0) - _F(5.0) * z2),
             (_F(1.4453057213202769) * z) * (x2 - y2),
             (_F(0.59004358992664352) * x) * (-x2 + _F(3.0) * y2)]
        return np.stack(o, 1).astype(np.float16).astype(np.float64)


# ---- exact forward ---------------------------------------------------------------------------------------------------
def _f16(v: np.ndarray) -> np.ndarray:
    with np.errstate(over="ignore", invalid="ignore"):
        return np.asarray(v, np.float64).astype(np.float16).astype(np.float64)


def _relu(v: np.ndarray) -> np.ndarray:
    return np.where(v > 0, v, 0.0)  # NaN -> 0


def _matmul(x: np.ndarray, W: np.ndarray) -> np.ndarray:
    """x @ W.T in float64 with IEEE semantics for non-finite inputs (0 * inf = NaN), which BLAS does not promise."""
    out = np.empty((x.shape[0], W.shape[0]))
    bad = ~np.isfinite(x).all(1)
    out[~bad] = x[~bad] @ W.T
    if bad.any():
        with np.errstate(invalid="ignore", over="ignore"):
            out[bad] = (x[bad][:, None, :] * W[None, :, :]).sum(-1)
    return out


def forward_exact(ws, feat: np.ndarray, sh: np.ndarray):
    """(density outputs [n, 16], nsb_inference rows [n, 16]) as fp16 values in float64: every layer's sum is exact (see certificate),
    so its fp16 value is the round-to-nearest of the float64 sum (+-inf past 65504)."""
    h1 = _relu(_f16(_matmul(feat, ws[0])))
    d = _f16(_matmul(h1, ws[1]))
    h2 = _relu(_f16(_matmul(np.concatenate([d, sh], 1), ws[2])))
    h3 = _relu(_f16(_matmul(h2, ws[3])))
    rgb = _f16(_matmul(h3, ws[4]))
    rgb[:, 3] = d[:, 0]  # extract_density
    return d, rgb


def _layers(ws, feat, sh):
    """(W, input) of the five layers, exact forward."""
    h1 = _relu(_f16(_matmul(feat, ws[0])))
    d = _f16(_matmul(h1, ws[1]))
    x3 = np.concatenate([d, sh], 1)
    h2 = _relu(_f16(_matmul(x3, ws[2])))
    h3 = _relu(_f16(_matmul(h2, ws[3])))
    return [(ws[0], feat), (ws[1], h1), (ws[2], x3), (ws[3], h2), (ws[4], h3)]


def _is_multiple(v: np.ndarray, u: float) -> bool:
    q = v / u
    return bool(np.all(q == np.round(q)))


def certificate(ws, feat, sh, units, skip=None, n_layers=5) -> float:
    """Asserts that every layer sum of every finite row is exact in fp16 in any summation order; returns the largest sum |w x| / (2048 u).
    units[l] = (ux, uw): the inputs of layer l that meet a non-zero weight are multiples of ux, its weights of uw, so every product is a
    multiple of u = ux uw. skip[l]: output indices of layer l left out (the overflow unit). n_layers: check the first n_layers only."""
    worst = 0.0
    for l, (W, x) in enumerate(_layers(ws, feat, sh)[:n_layers]):
        x = x[np.isfinite(x).all(1)]
        ux, uw = units[l]
        used = (W != 0).any(0)
        assert _is_multiple(x[:, used], ux) and _is_multiple(W, uw), f"layer {l + 1}: a product is not a multiple of its unit"
        mag = np.abs(x) @ np.abs(W).T
        if skip and l in skip:
            mag[:, skip[l]] = 0.0
        assert mag.max(initial=0.0) <= 65504.0, f"layer {l + 1}: a partial sum can overflow"
        r = mag.max(initial=0.0) / (2048.0 * ux * uw)
        assert r <= 1.0, f"layer {l + 1}: sum |w x| = {mag.max()} exceeds 2048 units"
        worst = max(worst, r)
    return worst


# ---- the model families -----------------------------------------------------------------------------------------------
N_INT_MODELS = 32  # 4 strides x 8 cyclic shifts of a sparsity pattern: every weight is non-zero in four of them


def _mask(n_out, n_in, shift, stride, period=8):
    i, j = np.meshgrid(np.arange(n_out), np.arange(n_in), indexing="ij")
    return ((stride * i + j + shift) % period) == 0


def integer_table(seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    return rng.integers(-2, 3, (N_LEVELS, ENTRIES, 2)).astype(np.float64)


def integer_weights(m: int, seed: int = 0):
    """Model m of the family: W1..W5 with the pattern of stride 1 + 2 * (m // 8) shifted by m % 8, entries in {-2, -1, 1, 2} (W2) or {-1, 1}, W3's SH
    columns zero."""
    rng = np.random.default_rng(1000 + seed * 97 + m)
    ws = []
    for l, (o, i) in enumerate(SHAPES):
        mask = _mask(o, i, m % 8, 1 + 2 * (m // 8))
        if l == 2:
            mask[:, 16:] = False
        vals = np.array([-2.0, -1.0, 1.0, 2.0]) if l == 1 else np.array([-1.0, 1.0])  # sums grow with depth: keep them under 2048
        p = [0.25, 0.75] if l == 3 else None  # W4 reads ReLU outputs only: mostly positive rows keep every L4 unit live on some rows
        ws.append(rng.choice(vals, (o, i), p=p) * mask)
    return ws


N_SH_MODELS = 64  # 16 column shifts x 2 halves of W3 x 2 routings: every SH weight of W3 reaches an output in one of them


def sh_weights(k: int, dens_ws):
    """SH probe k = m + 16 * half + 32 * route: the density MLP of dens_ws; W3 row j = 2 * (+-1) at SH column (j + m) % 16, + on rows
    j % 32 < 16 and on the constant column 0, - on the others, so rows j and j + 16 hold relu(2 sh) and relu(-2 sh); W4 the cyclic
    permutation by k; W5 row r (r != 3) = 0.5 * (the + unit - the - unit) of SH column (r + 8 * route) % 16 from rows
    32 * half .. 32 * half + 31; one of the two terms is 0, so every output is that column's fp16 SH value exactly (column 0: both units
    hold 2 sh0 > 0, 0.25 each, and sh0 / 2 is a normal fp16 value)."""
    m, half, route = k % 16, (k // 16) % 2, k // 32
    j = np.arange(64)
    col = (j + m) % 16
    sign = np.where(j % 32 < 16, 1.0, -1.0)
    sign[col == 0] = 1.0
    W3 = np.zeros((64, 32))
    W3[j, 16 + col] = 2.0 * sign
    W4 = np.zeros((64, 64))
    W4[j, (j + k) % 64] = 1.0  # h3[i] = relu(h2[(i + k) % 64]): the 64 probes put a one on every weight of W4
    W5 = np.zeros((16, 64))
    for r in range(16):
        if r == 3:
            continue
        c = (r + 8 * route) % 16
        plus = 32 * half + (c - m) % 16  # the + unit of column c in this half, then its - partner
        # column 0 (the constant SH0 > 0): both units hold relu(2 sh0), 0.25 each
        W5[r, (plus - k) % 64] = 0.25 if c == 0 else 0.5
        W5[r, (plus + 16 - k) % 64] = 0.25 if c == 0 else -0.5
    return [dens_ws[0], dens_ws[1], W3, W4, W5]


def scaled(ws, table, s_table=0, s=(0, 0, 0, 0, 0)):
    return [w * 2.0 ** e for w, e in zip(ws, s)], table * 2.0 ** s_table


def units_of(s_table=0, s=(0, 0, 0, 0, 0)):
    """(input unit, weight unit) of the five layers of a scaled integer model: features 2^s_table, weights 2^s[l]; each layer's outputs
    are multiples of the product of the two."""
    out, ux = [], 2.0 ** s_table
    for e in s:
        out.append((ux, 2.0 ** e))
        ux *= 2.0 ** e
    return out


RANGE_MODELS = {
    # name: (integer model, table exponent, W1..W5 exponents)
    "subnormal": (3, -20, (0, -4, 8, 0, -8)),  # features 2^-20.., density and rgb outputs multiples of 2^-24, hidden values subnormal
    "top": (2, 0, (0, 9, -9, 0, 5)),           # density outputs multiples of 512, rgb outputs of 32, into the top fp16 binades
    "overflow": (1, 0, (0, 0, 0, 0, 0)),       # plus OVERFLOW_UNIT: see overflow_model
}
OVERFLOW_UNIT, OVERFLOW_FEATURE = 5, 6  # L1 unit 5 = 2^15 * feature 6 (level 3, feature 0); W2's column 5 is zero


def range_model(name: str):
    """(ws, table, units, skip) of a range model."""
    m, st, s = RANGE_MODELS[name]
    ws, table = scaled(integer_weights(m), integer_table(m), st, s)
    skip = None
    if name == "overflow":
        ws[0][OVERFLOW_UNIT] = 0.0
        ws[0][OVERFLOW_UNIT, OVERFLOW_FEATURE] = 2.0 ** 15  # feature 2 -> 65536 -> inf, feature 1 -> 32768, <= 0 -> 0 after ReLU
        ws[1][:, OVERFLOW_UNIT] = 0.0                       # every successor sees 0 * h: 0, or NaN where h = inf
        skip = {0: [OVERFLOW_UNIT]}                         # one term: exact, then one rounding to fp16 in either policy
    return ws, table, units_of(st, s), skip


def exact_models():
    """name -> (params, ws, table, units, skip) of every exact model: the integer family, the SH probes, the range models."""
    out = {}
    for m in range(N_INT_MODELS):
        ws, t = integer_weights(m), integer_table(m)
        out[f"int{m}"] = (ws, t, units_of(), None)
    for k in range(N_SH_MODELS):
        ws, t = sh_weights(k, integer_weights(k % N_INT_MODELS)), integer_table(k % N_INT_MODELS)
        out[f"sh{k}"] = (ws, t, None, None)
    for name in RANGE_MODELS:
        out[name] = range_model(name)
    return {k: (pack(v[0], v[1]),) + v for k, v in out.items()}


def exact_rows(n: int, seed: int):
    """(coords [n + 9, 7], kxyz [n, 3]): lattice rows, then the nine non-finite position rows."""
    k, d = lattice_rows(n, seed)
    c = np.concatenate([lattice_coords(k, d), nonfinite_coords(d)])
    return c, k


def exact_reference(ws, table, coords: np.ndarray, kxyz: np.ndarray):
    """(features [N, 32], density outputs [N, 16], inference rows [N, 16]) for exact_rows: NaN features on the non-finite rows."""
    feat = np.full((coords.shape[0], 32), np.nan)
    feat[: kxyz.shape[0]] = table_features(table, kxyz)
    sh = sh4_f32(coords[:, 4:])
    d, rgb = forward_exact(ws, feat, sh)
    return feat, d, rgb


def mismatch(got_bits: np.ndarray, want: np.ndarray) -> np.ndarray:
    """bool mask: the fp16 values (bits) differ from want (float64 fp16 values); NaN matches NaN, +0 matches -0."""
    v = np.asarray(got_bits, np.uint16).view(np.float16).astype(np.float64)
    return ~((v == want) | (np.isnan(v) & np.isnan(want)))


# ---- rows ---------------------------------------------------------------------------------------------------------------
def lattice_rows(n: int, seed: int, outside: bool = True):
    """(kxyz [n, 3], dirs [n, 3]): lattice coordinates mostly inside [0, 16], some far outside the cube; random directions with the
    six axis directions, the zero direction (0.5, 0.5, 0.5) and components outside [0, 1] among them."""
    rng = np.random.default_rng(seed)
    k = rng.integers(0, 17, (n, 3))
    if outside:
        far = rng.random(n) < 0.1
        k[far] = rng.integers(-40, 60, (int(far.sum()), 3))
        k[:4] = [[-1, 0, 0], [17, 16, 16], [-1000, 5, 3000], [2 ** 20, -(2 ** 20), 7]]
    d = rng.random((n, 3)).astype(np.float32)
    special = np.array([[1, .5, .5], [0, .5, .5], [.5, 1, .5], [.5, 0, .5], [.5, .5, 1], [.5, .5, 0], [.5, .5, .5],
                        [1.7, -0.4, 0.5], [-2.0, 3.0, 0.25], [0.5, 0.5, 7.0]], np.float32)
    d[4:4 + len(special)] = special
    return k, d


def nonfinite_coords(dirs: np.ndarray) -> np.ndarray:
    """Rows whose position has a NaN or +-inf component (the other components on the lattice)."""
    vals = np.array([np.nan, np.inf, -np.inf], np.float32)
    rows = []
    for a in range(3):
        for v in vals:
            p = lattice_x(np.array([3, 8, 12]))
            p[a] = v
            rows.append(p)
    c = np.zeros((len(rows), 7), np.float32)
    c[:, :3] = rows
    c[:, 3] = 0.01
    c[:, 4:] = dirs[: len(rows)]
    return c


# ---- coverage -----------------------------------------------------------------------------------------------------------
def coverage(models) -> list:
    """models: [(ws, feat, sh)]. Returns the list of 5 bool matrices: weight (l, o, i) is covered when, in some model where it is
    non-zero, some row has a non-zero input i and output o of layer l reaches a network output through live ReLUs (a non-zero
    derivative of some output with respect to that layer's pre-activation o). Changing that weight alone then changes an output."""
    cov = [np.zeros(s, bool) for s in SHAPES]
    for ws, feat, sh in models:
        fin = np.isfinite(feat).all(1)
        feat, sh = feat[fin], sh[fin]
        L = _layers(ws, feat, sh)
        pre = [_matmul(x, W) for W, x in L]
        live = [(_f16(p) > 0).astype(np.float64) for p in pre]
        # derivatives of the 32 outputs (16 density, 16 inference rows with row 3 = density 0) w.r.t. each layer's pre-activation
        n = feat.shape[0]
        g = [None] * 5
        g5 = np.zeros((n, 32, 16))
        g5[:, 16 + np.array([r for r in range(16) if r != 3]), [r for r in range(16) if r != 3]] = 1.0
        g[4] = g5
        g[3] = (g[4] @ ws[4]) * live[3][:, None, :]
        g[2] = (g[3] @ ws[3]) * live[2][:, None, :]
        g2 = np.zeros((n, 32, 16))
        g2[:, np.arange(16), np.arange(16)] = 1.0
        g2[:, 16 + 3, 0] = 1.0
        g2 += (g[2] @ ws[2])[:, :, :16]
        g[1] = g2
        g[0] = (g[1] @ ws[1]) * live[0][:, None, :]
        for l, (W, x) in enumerate(L):
            reach = (np.abs(g[l]).sum(1) > 0)  # [n, out]
            inp = x != 0                         # [n, in]
            hit = (reach.T.astype(np.int64) @ inp.astype(np.int64)) > 0
            cov[l] |= hit & (W != 0)
    return cov


# ---- interval forward ----------------------------------------------------------------------------------------------------
def f16_down(v: np.ndarray) -> np.ndarray:
    h = _f16(v)
    return np.where(h > v, np.nextafter(h.astype(np.float16), np.float16(-np.inf)).astype(np.float64), h)


def f16_up(v: np.ndarray) -> np.ndarray:
    h = _f16(v)
    return np.where(h < v, np.nextafter(h.astype(np.float16), np.float16(np.inf)).astype(np.float64), h)


def _ilayer(W, lo, hi, acc16: bool, relu: bool):
    Wp, Wn = np.maximum(W, 0.0), np.minimum(W, 0.0)
    mag_x = np.maximum(np.abs(lo), np.abs(hi))
    if not acc16:
        slo = lo @ Wp.T + hi @ Wn.T
        shi = hi @ Wp.T + lo @ Wn.T
        err = (W.shape[1] * EPS32 + 2.0 ** -40) * (mag_x @ np.abs(W).T)
        ylo, yhi = f16_down(slo - err), f16_up(shi + err)
    else:
        ylo = np.zeros((lo.shape[0], W.shape[0]))
        yhi = np.zeros_like(ylo)
        for k0 in range(0, W.shape[1], 16):
            s = slice(k0, k0 + 16)
            plo = lo[:, s] @ Wp[:, s].T + hi[:, s] @ Wn[:, s].T
            phi = hi[:, s] @ Wp[:, s].T + lo[:, s] @ Wn[:, s].T
            err = (EPS16 + 2.0 ** -40) * (np.maximum(np.abs(ylo), np.abs(yhi)) + mag_x[:, s] @ np.abs(W[:, s]).T)
            ylo, yhi = f16_down(ylo + plo - err), f16_up(yhi + phi + err)
    if relu:
        ylo, yhi = np.maximum(ylo, 0.0), np.maximum(yhi, 0.0)
    return ylo, yhi


def forward_interval(ws, feat: np.ndarray, sh: np.ndarray, acc16: bool):
    """(lo, hi), each [n, 32]: columns 0-15 the density outputs, 16-31 the nsb_inference rows (row 3 = density 0). Finite features."""
    lo, hi = _ilayer(ws[0], feat, feat, acc16, True)
    dlo, dhi = _ilayer(ws[1], lo, hi, acc16, False)
    lo, hi = _ilayer(ws[2], np.concatenate([dlo, sh], 1), np.concatenate([dhi, sh], 1), acc16, True)
    lo, hi = _ilayer(ws[3], lo, hi, acc16, True)
    rlo, rhi = _ilayer(ws[4], lo, hi, acc16, False)
    rlo[:, 3], rhi[:, 3] = dlo[:, 0], dhi[:, 0]
    return np.concatenate([dlo, rlo], 1), np.concatenate([dhi, rhi], 1)


def width_ulps(lo: np.ndarray, hi: np.ndarray) -> np.ndarray:
    """[n, 32]: hi - lo in fp16 ulps of each output's scale, the largest |value| the output's intervals reach over the batch (near
    zero an ulp of the value itself says nothing about the arithmetic that produced it)."""
    scale = np.maximum(np.maximum(np.abs(lo), np.abs(hi)).max(0), 2.0 ** -14)
    return (hi - lo) / np.spacing(scale.astype(np.float16)).astype(np.float64)[None]


def outside(got_bits: np.ndarray, lo: np.ndarray, hi: np.ndarray) -> np.ndarray:
    """bool mask: the fp16 value (bits) lies outside [lo, hi] or is NaN."""
    v = np.asarray(got_bits, np.uint16).view(np.float16).astype(np.float64)
    return ~((v >= lo) & (v <= hi))


def random_model(seed: int, gain: float) -> np.ndarray:
    """A fox-geometry parameter block (encoding_domain.make_model) with its MLP weights scaled by `gain`."""
    from encoding_domain import GEOMETRIES, make_model

    p = make_model(GEOMETRIES["fox"], seed).copy()
    w = p[:N_MLP].view(np.float16).astype(np.float64) * gain
    p[:N_MLP] = w.astype(np.float16).view(np.uint16)
    return p


def random_rows(n: int, seed: int) -> np.ndarray:
    """NerfCoordinate rows: random positions and directions in [0, 1], with the encoding-domain position classes (outside the cube,
    lattice points, +-1e6) mixed in, finite only."""
    from encoding_domain import GEOMETRIES, coord_rows, level_geometry, positions

    rng = np.random.default_rng(seed)
    c = np.zeros((n, 7), np.float32)
    c[:, :3] = rng.random((n, 3), dtype=np.float32)
    c[:, 3] = 0.01
    c[:, 4:] = rng.random((n, 3), dtype=np.float32)
    dom = coord_rows(positions(*level_geometry(GEOMETRIES["fox"])), seed=seed, specials=False)
    k = min(n // 4, dom.shape[0])
    c[:k] = dom[:k]
    out = rng.random(n) < 0.05
    c[out, :3] = rng.uniform(-1.5, 2.5, (int(out.sum()), 3)).astype(np.float32)
    return c
