"""The fully fused MLPs on the H100 over their operand space, against the float64 reference (tests/network_reference.py), through the
C ABI, under both accumulator policies (NSB_MLP_ACC_F16 and NSB_MLP_ACC_F32):
  * every exact model (every weight of W1..W5 reaches an output in one of them) on nsb_density and nsb_inference, all 16 output rows,
    bit for bit (NaN as NaN, +0 as -0), and the range models against the oracle too;
  * batch shapes up to the grid-stride loop's later waves and padded strides: every padding column is the network on zero features and the
    zero direction, nothing is written past 16 x n_padded, and a side stream computes what the default stream does;
  * random models (the fox model and two wider-gain seeds): every output of every row inside its interval;
  * the other consumers of the tile loop and the backward wgmma: nsb_density_on_grid (with the density-grid filter), nsb_rgba_on_grid and
    nsb_density_gradient's density and dL/dfeatures, exact on integer models;
  * the accumulators' rounding (direction, ties, per-instruction rounding, internal precision) on designed sub-ulp sums;
  * the argument checks of n_padded, and the tile loop's 32-bit bound: nsb_density_gradient at n_padded = 2^32 - 128."""
import ctypes as C
import time

import numpy as np
import pytest

import network_reference as nr
from nerfshop_b200 import abi
from nerfshop_b200 import synthetic as syn
from oracle import oracle as orc

pytestmark = pytest.mark.gpu

POLICIES = {"f16": abi.NSB_MLP_ACC_F16, "f32": abi.NSB_MLP_ACC_F32}
ORACLE_POLICY = {abi.NSB_MLP_ACC_F16: 1, abi.NSB_MLP_ACC_F32: 0}
SENTINEL = 0x7D5A  # a NaN payload no kernel writes
GUARD = 4096       # halves after 16 x n_padded that must stay untouched


@pytest.fixture(scope="module")
def r(built_lib):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nerfshop_b200.renderer import NerfRenderer

    rr = NerfRenderer(0)
    yield rr
    rr.set_mlp_accumulator(abi.NSB_MLP_ACC_F16)
    rr.close()


@pytest.fixture(scope="module")
def models():
    return nr.exact_models()


@pytest.fixture(scope="module")
def rows():
    return nr.exact_rows(2048, seed=3)


def _upload(r, params, desc=None):
    r.upload_model(desc or nr.desc(), params)


def _net(r, fn, coords_dev, n, n_pad, stream=None):
    """fn's [16, n_pad] output (uint16) in a sentinel-filled buffer; asserts the guard after it is untouched."""
    import torch

    out = torch.full((16 * n_pad + GUARD,), SENTINEL, dtype=torch.int16, device="cuda")
    s = stream.cuda_stream if stream is not None else None
    st = fn(r.ctx, coords_dev.data_ptr() if coords_dev is not None else None, n, out.data_ptr(), n_pad, s)
    assert st == abi.NSB_OK, r.lib.nsb_last_error()
    torch.cuda.synchronize()
    h = out.cpu().numpy().view(np.uint16)
    assert (h[16 * n_pad:] == SENTINEL).all(), "written past 16 x n_padded"
    return h[: 16 * n_pad].reshape(16, n_pad)


def _dev(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("policy", sorted(POLICIES))
def test_exact_models_bit_for_bit(r, models, rows, policy):
    coords, k = rows
    n = coords.shape[0]
    n_pad = (n + 127) // 128 * 128
    c = _dev(coords)
    r.set_mlp_accumulator(POLICIES[policy])
    old = orc.set_mlp_policy(ORACLE_POLICY[POLICIES[policy]])
    try:
        for name, (params, ws, table, _, _) in models.items():
            _upload(r, params)
            feat, d, rgb = nr.exact_reference(ws, table, coords, k)
            if name == "int0":  # the premise: lattice features are table entries, NaN for non-finite positions
                enc = r.encode(coords).T.view(np.float16).astype(np.float64)
                assert np.array_equal(enc[: k.shape[0]], feat[: k.shape[0]]) and np.isnan(enc[k.shape[0]:]).all()
            got_d = _net(r, r.lib.nsb_density, c, n, n_pad)[:, :n].T
            got = _net(r, r.lib.nsb_inference, c, n, n_pad)[:, :n].T
            bad_d, bad = nr.mismatch(got_d, d), nr.mismatch(got, rgb)
            assert not bad_d.any(), f"{name}: nsb_density (row, output) {np.argwhere(bad_d)[:4].tolist()}"
            assert not bad.any(), f"{name}: nsb_inference (row, output) {np.argwhere(bad)[:4].tolist()}"
            if name in nr.RANGE_MODELS:
                o = orc.Oracle(nr.desc(), params, None)
                assert not nr.mismatch(got_d, o.inference(coords, density_only=True).T.view(np.float16).astype(np.float64)).any()
                assert not nr.mismatch(got, o.inference(coords).T.view(np.float16).astype(np.float64)).any()
    finally:
        orc.set_mlp_policy(old)


def _wave():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count * 5 * 128  # tile_ctas' cap: 5 one-tile CTAs per SM


def _batch_sizes():
    return [0, 1, 127, 128, 129, 4913, 3 * _wave() + 77, 1_000_003]


@pytest.fixture(scope="module")
def big_rows():
    """The largest batch's lattice rows and the SH probe's reference on them (the smaller batches are its prefixes)."""
    n = max(_batch_sizes())
    k, d = nr.lattice_rows(n, seed=17)
    coords = nr.lattice_coords(k, d)
    ws = nr.sh_weights(5, nr.integer_weights(5))
    table = nr.integer_table(5)
    feat, sh = nr.table_features(table, k), nr.sh4_f32(d)
    nr.certificate(ws, feat, sh, nr.units_of(), n_layers=2)  # the density MLP is an integer model's; the rgb MLP a probe's
    dens, rgb = nr.forward_exact(ws, feat, sh)
    pd, prgb = nr.forward_exact(ws, np.zeros((1, 32)), nr.sh4_f32(np.full((1, 3), 0.5, np.float32)))
    assert (prgb[0] != 0).sum() >= 2  # the padding's rgb outputs are not all zero: the check sees them
    return coords, nr.pack(ws, table), dens, rgb, pd[0], prgb[0]


@pytest.mark.parametrize("policy", sorted(POLICIES))
def test_batch_shapes_padding_and_streams(r, big_rows, policy):
    import torch

    coords, params, dens, rgb, pad_d, pad_rgb = big_rows
    r.set_mlp_accumulator(POLICIES[policy])
    _upload(r, params)
    c_all = _dev(coords)
    side = torch.cuda.Stream()
    for n in _batch_sizes():
        base = (max(n, 1) + 127) // 128 * 128
        for n_pad in (base, base + 384):
            c = c_all[:n] if n else c_all[:1]
            for fn, want, pad in ((r.lib.nsb_density, dens, pad_d), (r.lib.nsb_inference, rgb, pad_rgb)):
                got = _net(r, fn, c, n, n_pad)
                bad = nr.mismatch(got[:, :n].T, want[:n])
                assert not bad.any(), f"n {n} n_padded {n_pad}: (row, output) {np.argwhere(bad)[:4].tolist()}"
                badp = nr.mismatch(got[:, n:].T, np.broadcast_to(pad, (n_pad - n, 16)))
                assert not badp.any(), f"n {n} n_padded {n_pad}: padding column {n + np.argwhere(badp)[0, 0]} is not the network on the zero input"
                if n in (129, 3 * _wave() + 77):
                    assert np.array_equal(_net(r, fn, c, n, n_pad, stream=side), got), "the side stream differs from the default stream"


@pytest.mark.parametrize("policy", sorted(POLICIES))
def test_random_models_inside_their_intervals(r, policy):
    """The fox model and two wider-gain seeds, 200,000 rows each (random rows with the encoding domain's position classes, out of the
    cube included): every one of the 32 outputs of every row lies inside its interval."""
    desc = syn.model_desc()
    acc16 = POLICIES[policy] == abi.NSB_MLP_ACC_F16
    r.set_mlp_accumulator(POLICIES[policy])
    models = {"fox": syn.make_model(seed=1337).params, "seed7_gain1.6": nr.random_model(7, 1.6), "seed8_gain2": nr.random_model(8, 2.0)}
    for i, (name, params) in enumerate(models.items()):
        coords = nr.random_rows(200_000, seed=31 + i)
        _upload(r, params, desc)
        o = orc.Oracle(desc, params, None)
        enc = o.encode(coords)
        assert np.array_equal(r.encode(coords), enc)  # the features the intervals start from are the device's
        ws, _ = nr.unpack(params)
        lo, hi = nr.forward_interval(ws, enc.T.view(np.float16).astype(np.float64), nr.sh4_f32(coords[:, 4:]), acc16)
        got = np.concatenate([r.density(coords).T, r.inference(coords).T], 1)
        out = nr.outside(got, lo, hi)
        w = nr.width_ulps(lo, hi).max(0)
        print(f"\n{name} {policy}: interval width per output (fp16 ulps of its scale), max over rows: {np.ceil(w).astype(int).tolist()}")
        assert not out.any(), f"{name}: {out.sum()} outputs outside their interval, (row, output) {np.argwhere(out)[:4].tolist()}"
        assert w[:16].max() <= nr.WIDTH_CAP[0] and w[16:].max() <= nr.WIDTH_CAP[1]


# (W2 row: weights on h1_0, h1_1, h1_2, h1_16), the float64 sum, its fp16 value after one round-to-nearest-even, after one per K=16 chunk
ROUNDING_PROBES = [
    ((2048, 1, 0.5, 0), 2049.5, 2050, 2050),            # direction: RZ would give 2048
    ((2048, 1, 0, 0), 2049, 2048, 2048),                # tie to even
    ((2048, 2, 1, 0), 2051, 2052, 2052),                # tie to even, upwards
    ((2048, 1, 2.0 ** -10, 0), 2049 + 2.0 ** -10, 2050, 2050),  # a 2^-21 relative fraction inside one chunk survives: fp32 level
    ((-2048, -1, -0.5, 0), -2049.5, -2050, -2050),      # symmetric
    ((2048, 1, 0, 1), 2050, 2050, 2048),                # chunk 0 = 2049 -> 2048, then + 1 = 2049 -> 2048: one rounding per instruction
    ((1024, 0.5, 0.25, 0), 1024.75, 1025, 1025),
]


@pytest.mark.parametrize("policy", sorted(POLICIES))
def test_accumulator_rounding_characterised(r, policy):
    """The rounding the interval reference allows for, measured: L1 passes features 0-2 and 16 (all 1) through, L2 row k sums them with
    designed sub-ulp fractions. fp32 accumulators round the exact sum once to nearest even; fp16 accumulators (m64nNk16 with an fp16 D)
    round to nearest even after every K=16 instruction and keep a 2^-10 fraction of a 2049 sum inside one instruction (a relative
    error below 2^-21, inside EPS16). A 2^-14 fraction (below fp32's 24 bits at 2049) is printed, not asserted."""
    ws = [np.zeros(s) for s in nr.SHAPES]
    ws[0][np.arange(32), np.arange(32)] = 1.0
    for k, (w, _, _, _) in enumerate(ROUNDING_PROBES + [((2048, 1, 2.0 ** -14, 0), 0, 0, 0)]):
        ws[1][k, [0, 1, 2, 16]] = w
    table = np.zeros((nr.N_LEVELS, nr.ENTRIES, 2))
    table[0] = 1.0
    table[1, :, 0] = 1.0
    table[8, :, 0] = 1.0
    r.set_mlp_accumulator(POLICIES[policy])
    _upload(r, nr.pack(ws, table))
    coords = nr.lattice_coords(np.array([[1, 2, 3], [9, 0, 16]]), np.full((2, 3), 0.5, np.float32))
    got = r.density(coords).view(np.float16).astype(np.float64)
    chunked = POLICIES[policy] == abi.NSB_MLP_ACC_F16
    for k, (_, exact, once, per_chunk) in enumerate(ROUNDING_PROBES):
        assert (got[k] == (per_chunk if chunked else once)).all(), f"probe {k}: sum {exact} gave {got[k].tolist()}"
    print(f"\n{policy}: 2049 + 2^-14 in one instruction -> {got[len(ROUNDING_PROBES), 0]:g} (2050: more than 24 bits kept inside)")


# ---- the other consumers of the tile loop -------------------------------------------------------------------------------
TRAIN = (0.25, 0.75)  # train AABB of extent 2^-1: warping is exact


def _lattice_query(res, k0):
    """An NsbGridQuery whose grid point x (per axis) warps to (x + k0 - 0.5) / 16 exactly: spacing 1/32 in world units, the train AABB
    [0.25, 0.75]^3 of extent 1/2."""
    q = abi.NsbGridQuery()
    for a in range(3):
        rmin = np.float32(TRAIN[0] + (k0[a] - 0.5) / 32.0)
        q.res[a] = res[a]
        q.aabb_min[a] = float(rmin)
        q.aabb_max[a] = float(rmin + np.float32(res[a] / 32.0))
        q.train_aabb_min[a], q.train_aabb_max[a] = TRAIN
    return q


def _query_points(q, z0, z1):
    """(world positions [m, 3] float64, lattice k [m, 3]) of grid points with z in [z0, z1), x fastest."""
    rx, ry = q.res[0], q.res[1]
    z, y, x = np.meshgrid(np.arange(z0, z1), np.arange(ry), np.arange(rx), indexing="ij")
    g = np.stack([x.ravel(), y.ravel(), z.ravel()], 1)
    p = np.stack([np.float64(q.aabb_min[a]) + g[:, a] / 32.0 for a in range(3)], 1)
    k = np.rint((p - TRAIN[0]) * 32.0 + 0.5).astype(np.int64)
    assert np.array_equal((k - 0.5) / 32.0 + TRAIN[0], p)
    return p, k


def _mip_and_cell(p):
    """mip_from_pos and cascaded_grid_idx_at (nsb_device.cuh) for positions that are multiples of 2^-6 inside the cascades."""
    a = p - 0.5
    maxval = np.abs(a).max(1)
    e = np.frexp(maxval)[1]
    mip = np.where(maxval == 0, 1, np.clip(e + 1, 0, 4))
    cell = np.clip(np.trunc(a * 2.0 ** (7 - mip)[:, None] + 64.0), 0, 127).astype(np.uint32)
    return mip, syn.morton3d(cell[:, 0], cell[:, 1], cell[:, 2]).astype(np.int64)


@pytest.mark.parametrize("policy", sorted(POLICIES))
def test_density_on_grid_exact(r, models, policy):
    """512 x 256 x 128 grid points (about 200 waves of tiles) on lattice positions inside the five cascades, an integer model, a density
    grid of ones with cascade 2 and half of cascade 4 zeroed: the raw density where the grid is set, -10000 where it is not."""
    import torch

    params, ws, table, _, _ = models["int0"]
    r.set_mlp_accumulator(POLICIES[policy])
    _upload(r, params)
    grid = np.ones((5, 128 ** 3), np.float32)
    grid[2] = 0.0
    ix = np.arange(128)
    X, Y, Z = np.meshgrid(ix, ix, ix, indexing="ij")
    grid[4, syn.morton3d(X[X < 64], Y[X < 64], Z[X < 64])] = 0.0
    r.upload_density_grid(grid)
    res, k0 = (512, 256, 128), (-247, -119, -55)
    q = _lattice_query(res, k0)
    out = torch.empty(res[2] * res[1] * res[0], dtype=torch.float32, device="cuda")
    abi.check(r.lib, r.lib.nsb_density_on_grid(r.ctx, C.byref(q), out.data_ptr(), None), "nsb_density_on_grid")
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    n_filtered = 0
    for z0 in range(0, res[2], 4):
        p, k = _query_points(q, z0, z0 + 4)
        assert (np.abs(p - 0.5) < 8).all()
        feat = nr.table_features(table, k)
        h1 = np.maximum(feat @ ws[0].T, 0.0)
        assert (np.abs(feat) @ np.abs(ws[0]).T).max() <= 2048 and (h1 @ np.abs(ws[1][0])).max() <= 2048  # exact in fp16
        want = (h1 @ ws[1][0]).astype(np.float32)
        mip, cell = _mip_and_cell(p)
        empty = grid[mip, cell] < 0.01
        want[empty] = -10000.0
        n_filtered += int(empty.sum())
        sl = got[z0 * res[0] * res[1]:(z0 + 4) * res[0] * res[1]]
        bad = sl != want
        assert not bad.any(), f"z {z0}..: {bad.sum()} grid points differ, first {np.argwhere(bad)[:4].ravel().tolist()}"
    assert 0.05 < n_filtered / got.size < 0.95


@pytest.mark.parametrize("policy", sorted(POLICIES))
def test_rgba_on_grid_through_an_sh_probe(r, models, policy):
    """The launch-wide direction through an SH probe: rgb = fl(raw * a) bit for bit with the device's own a, raw = the probe's SH values,
    and a = 1 - __expf(-relu(d) / 100) within __expf's documented error (2 + floor(1.173 |x|) ulp) of the float64 value."""
    import torch

    params, ws, table, _, _ = models["sh5"]
    r.set_mlp_accumulator(POLICIES[policy])
    _upload(r, params)
    res, k0 = (128, 64, 32), (-60, -30, -10)
    q = _lattice_query(res, k0)
    ray = np.array([0.3, -0.5, 0.8], np.float32)
    ray /= np.float32(np.linalg.norm(ray))
    d = (C.c_float * 3)(*[float(v) for v in ray])
    out = torch.empty((res[2] * res[1] * res[0], 4), dtype=torch.float32, device="cuda")
    abi.check(r.lib, r.lib.nsb_rgba_on_grid(r.ctx, C.byref(q), d, abi.NSB_ACT_NONE, abi.NSB_ACT_RELU, out.data_ptr(), None), "nsb_rgba_on_grid")
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    _, k = _query_points(q, 0, res[2])
    dw = ((ray + np.float32(1.0)) * np.float32(0.5))[None]
    _, rgb = nr.forward_exact(ws, nr.table_features(table, k), np.repeat(nr.sh4_f32(dw), k.shape[0], 0))
    a = got[:, 3]
    np.testing.assert_array_equal(got[:, :3].view(np.uint32), (rgb[:, :3].astype(np.float32) * a[:, None]).view(np.uint32))
    x = (-np.maximum(rgb[:, 3], 0.0).astype(np.float32) / np.float32(100.0)).astype(np.float64)
    e = np.exp(x)
    want = np.clip(1.0 - e, 0.0, 1.0)
    tol = (3.0 + np.floor(1.173 * np.abs(x))) * np.spacing(e.astype(np.float32)).astype(np.float64) + 2.0 ** -24
    assert (np.abs(a - want) <= tol).all(), f"max |a - a64| / tol = {(np.abs(a - want) / tol).max()}"
    assert (rgb[:, 3] > 0).mean() > 0.2 and (a > 0).mean() > 0.2 and (got[:, :3] != 0).any()


@pytest.mark.parametrize("policy", sorted(POLICIES))
def test_density_gradient_forward_and_dfeat_exact(r, models, rows, policy):
    """nsb_density_gradient on integer models: the raw density and dL/dfeatures = 128 W1^T (relu'(h1) * W2[0, :]) exactly (every term
    is a multiple of 128 and the sums stay below 2048 of them). The position gradient is pinned by test_gpu_density_gradient.py."""
    import torch

    coords, k = rows
    coords, n = coords[: k.shape[0]], k.shape[0]
    n_pad = (n + 127) // 128 * 128
    r.set_mlp_accumulator(POLICIES[policy])
    c = _dev(coords)
    for name in ("int0", "int9", "int21", "subnormal"):
        params, ws, table, _, _ = models[name]
        _upload(r, params)
        feat = nr.table_features(table, k)
        h1 = nr._relu(nr._f16(feat @ ws[0].T))
        d0 = nr._f16(h1 @ ws[1][0])
        dfeat = ((h1 > 0) * (128.0 * ws[1][0])) @ ws[0]
        assert np.array_equal(nr._f16(dfeat), dfeat)
        grad = torch.zeros((n, 3), dtype=torch.float32, device="cuda")
        dens = torch.full((n_pad,), SENTINEL, dtype=torch.int16, device="cuda")
        df = torch.full((32, n_pad), SENTINEL, dtype=torch.int16, device="cuda")
        abi.check(r.lib, r.lib.nsb_density_gradient(r.ctx, c.data_ptr(), n, grad.data_ptr(), 3, dens.data_ptr(), df.data_ptr(), n_pad, None),
                  "nsb_density_gradient")
        torch.cuda.synchronize()
        assert not nr.mismatch(dens.cpu().numpy().view(np.uint16)[:n], d0).any(), name
        bad = nr.mismatch(df.cpu().numpy().view(np.uint16)[:, :n].T, dfeat)
        assert not bad.any(), f"{name}: dfeat (row, feature) {np.argwhere(bad)[:4].tolist()}"


def test_n_padded_argument_checks(r, models):
    import torch

    _upload(r, models["int0"][0])
    c = torch.zeros((256, 7), device="cuda")
    out = torch.zeros(16 * 512, dtype=torch.int16, device="cuda")
    for fn in (r.lib.nsb_density, r.lib.nsb_inference):
        assert fn(r.ctx, c.data_ptr(), 129, out.data_ptr(), 128, None) == abi.NSB_ERR_INVALID  # n_padded < n
        assert fn(r.ctx, c.data_ptr(), 100, out.data_ptr(), 200, None) == abi.NSB_ERR_INVALID  # not a multiple of 128
        assert fn(r.ctx, c.data_ptr(), 128, out.data_ptr(), 256, None) == abi.NSB_OK
    torch.cuda.synchronize()


def test_density_gradient_tile_loop_does_not_wrap_at_2_32(r, models):
    """nsb_density_gradient(n = 1, n_padded = 2^32 - 128) with no density or dfeat output: a 12-byte gradient and one coordinate row.
    The grid is capped at sm_count x ctas_per_sm CTAs, a stride of S = 84,480 rows on a 132-SM H100. A loop that steps a uint32 row base
    by S wraps once the base passes 2^32 - S, to a small base, and walks the rows again; 2^32 mod 84,480 = 4,096, so each wrap shifts the
    residue by 4,096 and about three CTAs in four never land in the exit window [n_padded, 2^32): that launch does not terminate. The
    tile loop walks tile indices (< 2^25, step < 2^16), which cannot wrap. A build with the row-base loop must never be run on this case."""
    import torch

    _upload(r, models["int0"][0])
    coords = nr.lattice_coords(np.array([[3, 8, 12]]), np.full((1, 3), 0.5, np.float32))
    c = _dev(coords)
    g_plain = torch.zeros((1, 3), dtype=torch.float32, device="cuda")
    abi.check(r.lib, r.lib.nsb_density_gradient(r.ctx, c.data_ptr(), 1, g_plain.data_ptr(), 3, None, None, 128, None), "plain")
    g = torch.zeros((1, 3), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    abi.check(r.lib, r.lib.nsb_density_gradient(r.ctx, c.data_ptr(), 1, g.data_ptr(), 3, None, None, (1 << 32) - 128, None), "2^32 - 128")
    torch.cuda.synchronize()
    print(f"\nnsb_density_gradient over 2^32 - 128 rows: {time.perf_counter() - t0:.2f} s")
    np.testing.assert_array_equal(g.cpu().numpy().view(np.uint32), g_plain.cpu().numpy().view(np.uint32))
