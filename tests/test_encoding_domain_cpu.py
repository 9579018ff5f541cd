"""CPU tests of the hash-grid encoding over its whole input domain (no GPU needed).

The product's own build_levels and grid_index (nsb_device.cuh) are compiled by nvcc for the host and compared with the oracle's
restatement of tiny-cuda-nn's grid_index, `% size` on the uint32 index, on every level of a table of geometries, for grid coordinates
that positions far outside [0,1]^3 reach (uint32 wrap-around from negative coordinates, saturated conversions). The oracle's float->int
conversion, its encoding against an independent numpy one, and the accepted model descriptions are pinned alongside."""
import ctypes as C
import itertools
import zlib

import numpy as np
import pytest

import encoding_domain as ed
from nerfshop_b200 import abi, synthetic as syn
from oracle import oracle as orc
from test_oracle_units import _numpy_encode

U32 = [0, 1, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE, 0xFFFFFFFF]


def _host_levels(d):
    L = d.n_levels
    res, size, hashed = (np.zeros(L, np.uint32) for _ in range(3))
    n, in_range = C.c_uint64(), C.c_int()
    st = ed.host_lib().host_levels(C.byref(d), res.ctypes.data, size.ctypes.data, hashed.ctypes.data, C.byref(n), C.byref(in_range))
    return st, res, size, hashed, n.value, bool(in_range.value)


def _axis_values(d, l, scale, res):
    """Grid coordinates of one level: the structured ones (lattice edges, uint32 extremes) and every coordinate (and +1) that the
    position classes of the GPU tests reach on this level."""
    r = int(res[l])
    structured = {0, 1, r - 1, r, r + 1, 2 * r} | set(U32)
    x = np.concatenate([ed.positions(*ed.level_geometry(d)), ed.SPECIALS])
    g = ed.grid_coords(x, scale[l])
    reached = set(int(a) for a in g) | set((int(a) + 1) & 0xFFFFFFFF for a in g)
    as_u32 = lambda v: np.array(sorted(a & 0xFFFFFFFF for a in v), np.uint32)
    return as_u32(structured), as_u32(reached)


def _triples(structured, reached, rng):
    """Every structured triple; every reached value on each axis against every pair of structured partners; random uint32 triples."""
    parts = [np.array(list(itertools.product(structured, structured, structured)), np.uint32)]
    pairs = np.array(list(itertools.product(structured, structured)), np.uint32)
    for a in range(3):
        t = np.empty((reached.size * pairs.shape[0], 3), np.uint32)
        t[:, a] = np.repeat(reached, pairs.shape[0])
        others = [b for b in range(3) if b != a]
        t[:, others] = np.tile(pairs, (reached.size, 1))
        parts.append(t)
    parts.append(rng.integers(0, 2**32, (4096, 3), dtype=np.uint64).astype(np.uint32))
    return np.ascontiguousarray(np.concatenate(parts))


@pytest.mark.parametrize("name", list(ed.GEOMETRIES))
def test_host_grid_index_equals_tcnn_rule(name):
    d = ed.GEOMETRIES[name]
    st, res, size, hashed, _, _ = _host_levels(d)
    assert st == 0
    scale, res_t, size_t, hashed_t = ed.level_geometry(d)
    assert (res == res_t).all() and (size == size_t).all() and (hashed.astype(bool) == hashed_t).all()
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    lib, olib = ed.host_lib(), orc.lib()
    for l in range(d.n_levels):
        g = _triples(*_axis_values(d, l, scale, res), rng)
        want = np.zeros(g.shape[0], np.uint32)
        assert olib.orc_grid_index(C.byref(d), l, g.ctypes.data, g.shape[0], want.ctypes.data) == 0
        assert (want < size[l]).all()
        for mode in ((1, 2) if hashed[l] else (0, 2)):
            got = np.zeros_like(want)
            assert lib.host_grid_index(C.byref(d), l, mode, 0, g.ctypes.data, g.shape[0], got.ctypes.data) == 0
            bad = np.nonzero(got != want)[0]
            assert bad.size == 0, f"{name} level {l} mode {mode}: {bad.size} of {g.shape[0]} indices differ, e.g. {g[bad[0]]} -> {got[bad[0]]} != {want[bad[0]]}"


@pytest.mark.parametrize("name", list(ed.GEOMETRIES))
def test_in_range_shortcut_is_exact_where_the_host_allows_it(name):
    """grid_index<MODE, true> (the fused renderer's one-subtraction modulo) equals tcnn's rule for every coordinate up to res, on models
    whose dense levels pass dense_in_range; models that fail it have a dense level where the shortcut would be wrong."""
    d = ed.GEOMETRIES[name]
    st, res, size, hashed, _, in_range = _host_levels(d)
    assert st == 0
    lib, olib = ed.host_lib(), orc.lib()
    fails = False
    for l in range(d.n_levels):
        if hashed[l]:
            continue
        r = int(res[l])
        ax = np.unique(np.concatenate([np.arange(0, min(r, 24) + 1), np.arange(max(0, r - 24), r + 1)])).astype(np.uint32)
        g = np.ascontiguousarray(np.array(list(itertools.product(ax, ax, ax)), np.uint32))
        want, got = np.zeros(g.shape[0], np.uint32), np.zeros(g.shape[0], np.uint32)
        assert olib.orc_grid_index(C.byref(d), l, g.ctypes.data, g.shape[0], want.ctypes.data) == 0
        assert lib.host_grid_index(C.byref(d), l, 0, 1, g.ctypes.data, g.shape[0], got.ctypes.data) == 0
        if in_range:
            assert (got == want).all(), f"{name} level {l}"
        fails |= bool((got != want).any())
    assert in_range or fails


def test_shortcut_is_wrong_outside_the_cube():
    """The example of the fox model: warped z = -0.04 (world z = -1.66). The one-subtraction rule leaves an index ~4.29e9 on level 0,
    tcnn's rule gives one below the level's 4096 entries."""
    d = ed.GEOMETRIES["fox"]
    scale, res, size, _ = ed.level_geometry(d)
    g = ed.grid_coords(np.array([0.5, 0.5, -0.04], np.float32), scale[0])
    g = np.ascontiguousarray(g.reshape(1, 3))
    want, fast, exact = (np.zeros(1, np.uint32) for _ in range(3))
    assert orc.lib().orc_grid_index(C.byref(d), 0, g.ctypes.data, 1, want.ctypes.data) == 0
    ed.host_lib().host_grid_index(C.byref(d), 0, 0, 1, g.ctypes.data, 1, fast.ctypes.data)
    ed.host_lib().host_grid_index(C.byref(d), 0, 0, 0, g.ctypes.data, 1, exact.ctypes.data)
    assert int(want[0]) == 3976 and int(exact[0]) == 3976
    assert int(fast[0]) >= int(size[0])  # the reason the renderer takes the shortcut only for in-range frames


def test_oracle_float_to_int_is_cvt_rzi_s32():
    l = orc.lib()
    cases = {float("nan"): 0, float("inf"): 2**31 - 1, -float("inf"): -2**31, 2.0**31: 2**31 - 1, 3e9: 2**31 - 1, 1e30: 2**31 - 1,
             -(2.0**31): -2**31, -3e9: -2**31, -1e30: -2**31, 2147483520.0: 2147483520, -2147483520.0: -2147483520,
             -2.75: -2, 2.75: 2, -0.5: 0, 0.0: 0, -0.0: 0, 16777217.0: 16777216}
    for v, want in cases.items():
        assert l.orc_f2i(v) == want, v
    xs = np.random.default_rng(4).standard_normal(5000).astype(np.float32) * np.float32(1e9)
    got = np.array([l.orc_f2i(float(v)) for v in xs], np.int64)
    assert (got == np.clip(np.trunc(xs.astype(np.float64)), -2.0**31, 2.0**31 - 1).astype(np.int64)).all()


@pytest.mark.parametrize("name", list(ed.GEOMETRIES))
def test_oracle_encode_equals_numpy_on_the_whole_domain(name):
    d = ed.GEOMETRIES[name]
    params = ed.make_model(d, seed=11)
    oracle = orc.Oracle(d, params, None)
    rows = ed.coord_rows(ed.positions(*ed.level_geometry(d)), seed=2)
    got = oracle.encode(rows)
    ref = _numpy_encode(None, rows, desc=d, grid=params[10240:].view(np.float16)).view(np.uint16)
    nan_got, nan_ref = np.isnan(got.view(np.float16)), np.isnan(ref.view(np.float16))
    assert (nan_got == nan_ref).all()
    assert (got[~nan_got] == ref[~nan_ref]).all(), f"{(got[~nan_got] != ref[~nan_ref]).sum()} of {got.size} feature halves differ"
    # inf and NaN coordinates make that row's features NaN on every level (the weights are NaN); finite rows are finite
    bad_row = ~np.isfinite(rows[:, :3]).all(axis=1)
    assert nan_got[:, bad_row].all() and not nan_got[:, ~bad_row].any()


def _n_params(lib_fn, d):
    n = C.c_uint64()
    st = lib_fn(C.byref(d), C.byref(n))
    return st, n.value


DOMAIN = {
    **{k: (True, v) for k, v in ed.GEOMETRIES.items()},
    "log2_1": (True, ed.desc(log2=1)),
    "log2_24": (True, ed.desc(log2=24)),
    "pls_1": (True, ed.desc(pls=1.0)),
    "base_2048_pls_1": (True, ed.desc(base=2048, pls=1.0)),
    "nan_pls": (False, ed.desc(pls=float("nan"))),
    "inf_pls": (False, ed.desc(pls=float("inf"))),
    "pls_below_1": (False, ed.desc(pls=0.9)),
    "pls_0": (False, ed.desc(pls=0.0)),
    "pls_negative": (False, ed.desc(pls=-2.0)),
    "log2_0": (False, ed.desc(log2=0)),
    "log2_25": (False, ed.desc(log2=25)),
    "base_0": (False, ed.desc(base=0, pls=2.0)),
    "scale_overflows_uint32": (False, ed.desc(base=16, pls=8.0)),  # level 15: 16 * 8^15 - 1 = 2^49
    "scale_2_31": (True, ed.desc(base=2**31, pls=1.0)),            # res 2^31 + 1: fits
    "scale_2_32": (False, ed.desc(base=2**32 - 1, pls=1.0)),       # float(2^32 - 1) - 1 rounds to 2^32: res would not fit
}


@pytest.mark.parametrize("name", list(DOMAIN))
def test_parameter_count_and_accepted_domain_agree(built_lib, name):
    accepted, d = DOMAIN[name]
    lib = abi.load_library()
    st_p, n_p = _n_params(lib.nsb_model_n_params, d)
    st_o, n_o = _n_params(orc.lib().orc_model_n_params, d)
    assert (st_p == abi.NSB_OK) == (st_o == 0), f"product status {st_p}, oracle status {st_o}"
    assert (st_p == abi.NSB_OK) == accepted
    if accepted:
        assert n_p == n_o
        _, _, _, _, entries = syn.level_table(d)
        assert n_p == 10240 + 2 * entries
        st_h, _, size, _, n_h, _ = _host_levels(d)
        assert st_h == 0 and n_h == entries and (size <= (1 << d.log2_hashmap_size)).all()
    else:
        assert _host_levels(d)[0] != 0
