"""CPU tests: the oracle's building blocks against independent numpy restatements and invariants
(SURVEY.md §8c(3): the reference ships no tests, so the pins are properties + golden files)."""
import ctypes as C

import numpy as np

from conftest import random_coords
from nerfshop_b200 import abi, synthetic as syn
from oracle import oracle as orc


def test_half_conversion_matches_ieee():
    l = orc.lib()
    rng = np.random.default_rng(1)
    xs = np.concatenate([rng.standard_normal(4000).astype(np.float32) * s for s in (1e-8, 1e-6, 1e-3, 1.0, 300.0, 60000.0)])
    xs = np.concatenate([xs, np.array([0.0, -0.0, 65504.0, 65519.9, 65520.0, 2.0 ** -24, 2.0 ** -25, 1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11], np.float32)])
    with np.errstate(over="ignore"):
        ref = xs.astype(np.float16).view(np.uint16)
    got = np.array([l.orc_f2h(float(v)) for v in xs], np.uint16)
    assert (got == ref).all()
    hs = np.arange(0, 0x7C00, 7, dtype=np.uint16)
    back = np.array([l.orc_h2f(int(h)) for h in hs], np.float32)
    assert (back == hs.view(np.float16).astype(np.float32)).all()


def test_morton_and_cell_index():
    l = orc.lib()
    rng = np.random.default_rng(2)
    for _ in range(200):
        x, y, z = (int(v) for v in rng.integers(0, 128, 3))
        m = l.orc_morton3D(x, y, z)
        # de-interleave
        dx = sum(((m >> (3 * b)) & 1) << b for b in range(7))
        dy = sum(((m >> (3 * b + 1)) & 1) << b for b in range(7))
        dz = sum(((m >> (3 * b + 2)) & 1) << b for b in range(7))
        assert (dx, dy, dz) == (x, y, z)
        assert int(syn.morton3d(np.array([x]), np.array([y]), np.array([z]))[0]) == m
    # cascade m covers the cube of side 2^m about 0.5: its centre cell is the same for every cascade
    for mip in range(5):
        assert l.orc_cascaded_grid_idx_at(0.5, 0.5, 0.5, mip) == l.orc_morton3D(64, 64, 64)
    # mip_from_pos: |p-0.5|max in [2^(k-2), 2^(k-1)) -> mip k (clamped), exact centre -> 1 (frexpf(0) quirk of the reference)
    assert l.orc_mip_from_pos(0.5, 0.5, 0.5) == 1
    assert l.orc_mip_from_pos(0.6, 0.5, 0.5) == 0
    assert l.orc_mip_from_pos(0.5, 0.99, 0.5) == 0
    assert l.orc_mip_from_pos(1.01, 0.5, 0.5) == 1
    assert l.orc_mip_from_pos(0.5, 0.5, -0.6) == 2
    assert l.orc_mip_from_pos(2.4, 0.5, 0.5) == 2
    assert l.orc_mip_from_pos(9.0, 0.5, 0.5) == 4


def test_sobol_jitter_properties():
    l = orc.lib()
    vals = np.array([l.orc_ld_random_val(0, i * 786433 & 0xFFFFFFFF) for i in range(4096)], np.float32)
    assert vals.min() >= 0.0 and vals.max() <= 1.0
    assert abs(vals.mean() - 0.5) < 0.03  # scrambled-Sobol first sample over seeds is ~uniform
    # the same (index, seed) is deterministic; stratification over the index for a fixed seed
    per_seed = np.array([l.orc_ld_random_val(i, 12345) for i in range(16)], np.float32)
    assert len(np.unique(np.floor(per_seed * 16))) == 16  # (0,4,2)-net property of a scrambled Sobol dimension
    off = (C.c_float * 2)()
    l.orc_pixel_offset(0, off)
    assert abs(off[0] - 0.5) < 1e-6 and abs(off[1] - 0.5) < 1e-6  # spp 0 -> pixel centres
    l.orc_pixel_offset(3, off)
    assert 0.0 <= off[0] < 1.0 and 0.0 <= off[1] < 1.0


def test_level_table_matches_survey_numbers():
    desc = syn.model_desc(4)
    L = desc.n_levels
    scale = np.zeros(L, np.float32)
    res = np.zeros(L, np.uint32)
    off = np.zeros(L, np.uint32)
    size = np.zeros(L, np.uint32)
    assert orc.lib().orc_level_table(C.byref(desc), scale.ctypes.data, res.ctypes.data, off.ctypes.data, size.ctypes.data) == 0
    # SURVEY.md §2b: fox (aabb_scale 4) -> b = 1.5157, dense levels 0-3 with 4096, 15632, 50656(?), 175616 entries
    assert abs(desc.per_level_scale - 1.5157166) < 1e-5
    assert list(size[:2]) == [4096, 15632] and size[3] == 175616
    assert (size[4:] == 1 << 19).all()
    n = C.c_uint64()
    assert orc.lib().orc_model_n_params(C.byref(desc), C.byref(n)) == 0
    assert n.value == 10240 + 13074912  # SURVEY.md §2b: 13,074,912 fp16 grid parameters
    s2, r2, o2, z2, total = syn.level_table(desc)
    assert (r2 == res).all() and (o2 == off).all() and (z2 == size).all() and total * 2 == 13074912
    assert np.allclose(s2, scale, rtol=1e-6)


def _f2i_rz_sat(v):
    """cvt.rzi.s32.f32 as uint32: truncation, NaN -> 0, saturation to the int range, then the two's-complement bits."""
    v = np.asarray(v, np.float64)
    v = np.where(np.isnan(v), 0.0, np.clip(v, -2.0 ** 31, 2.0 ** 31 - 1))
    return np.trunc(v).astype(np.int64).astype(np.uint32)


def _numpy_encode(model, coords, desc=None, grid=None):
    """Independent restatement of the tcnn hash grid in numpy: float32 weights, fp16 accumulation. Total on float32 inputs:
    coordinates wrap through uint32, the index is `% size` on the uint32 value, and hash vs. dense follows tcnn's uint32 stride."""
    desc = model.desc if desc is None else desc
    grid = (model.grid if grid is None else grid).reshape(-1, 2)
    scale, res, offset, size, _ = syn.level_table(desc)
    # take the level scales from the oracle (libm exp2f bits), everything else is recomputed here
    L = desc.n_levels
    sc = np.zeros(L, np.float32)
    tmp = [np.zeros(L, np.uint32) for _ in range(3)]
    assert orc.lib().orc_level_table(C.byref(desc), sc.ctypes.data, *[t.ctypes.data for t in tmp]) == 0
    x = coords[:, :3].astype(np.float32)
    out = np.zeros((32, x.shape[0]), np.float16)
    for l in range(L):
        with np.errstate(invalid="ignore", over="ignore"):
            p = np.float32(np.float64(sc[l]) * x.astype(np.float64) + 0.5)  # fma == exact product + add, one rounding
            g = np.floor(p)
            w = (p - g).astype(np.float32)
        g = _f2i_rz_sat(g)
        acc = np.zeros((x.shape[0], 2), np.float16)
        r, n = np.uint32(res[l]), int(size[l])
        stride, dim = 1, 0
        while dim < 3 and stride <= n:
            stride, dim = (stride * int(res[l])) & 0xFFFFFFFF, dim + 1
        hashed = n < stride
        for c in range(8):
            wt = np.ones(x.shape[0], np.float32)
            gi = []
            for d in range(3):
                if c & (1 << d):
                    wt = (wt * w[:, d]).astype(np.float32)
                    gi.append(g[:, d] + np.uint32(1))
                else:
                    wt = (wt * (np.float32(1.0) - w[:, d])).astype(np.float32)
                    gi.append(g[:, d])
            with np.errstate(over="ignore"):
                if hashed:
                    idx = gi[0] ^ (gi[1] * np.uint32(2654435761)) ^ (gi[2] * np.uint32(805459861))
                else:
                    idx = gi[0] + gi[1] * r + gi[2] * (r * r)  # uint32 arithmetic: wraps like tcnn's
            idx = idx % np.uint32(n)
            vals = grid[int(offset[l]) + idx.astype(np.int64)].astype(np.float32)
            with np.errstate(invalid="ignore", over="ignore"):
                prod = (wt[:, None] * vals).astype(np.float32).astype(np.float16)
                acc = (acc.astype(np.float64) + prod.astype(np.float64)).astype(np.float16)  # exact sum, one rounding
        out[2 * l], out[2 * l + 1] = acc[:, 0], acc[:, 1]
    return out


def test_encode_matches_independent_numpy(scene, oracle):
    model, _ = scene
    coords = random_coords(500, seed=3)
    got = oracle.encode(coords)
    ref = _numpy_encode(model, coords).view(np.uint16)
    assert (got == ref).all(), f"{(got != ref).sum()} of {got.size} feature halves differ"


def test_trilinear_weights_and_hash_formula(scene):
    model, _ = scene
    scale, res, offset, size, _ = syn.level_table(model.desc)
    # hashed levels: index formula vs brute force on a few lattice points (SURVEY.md §8c(3))
    for l in (4, 9, 15):
        for (x, y, z) in ((0, 0, 0), (1, 2, 3), (int(res[l]) - 1, 7, 11), (123, 456, 789)):
            h = ((x * 1) ^ ((y * 2654435761) & 0xFFFFFFFF) ^ ((z * 805459861) & 0xFFFFFFFF)) % int(size[l])
            assert 0 <= h < (1 << 19)
    w = np.random.default_rng(0).random((100, 3)).astype(np.float32)
    tot = np.zeros(100, np.float64)
    for c in range(8):
        t = np.ones(100, np.float64)
        for d in range(3):
            t *= w[:, d] if c & (1 << d) else 1 - w[:, d]
        tot += t
    assert np.allclose(tot, 1.0)


def test_inference_matches_numpy_mlp(scene, oracle):
    """fp16 weights/activations, wmma __half accumulator fragments (the running sum is rounded to fp16 after every k-chunk of 16: Appendix B, the
    oracle's default policy), fp16 rounding between layers."""
    model, _ = scene
    coords = random_coords(200, seed=4)
    enc = oracle.encode(coords).view(np.float16).astype(np.float64)  # [32, n]
    mlp = model.params[: syn.N_MLP_PARAMS].view(np.float16).astype(np.float64)
    W1, W2, W3, W4, W5 = (mlp[a:b].reshape(s) for a, b, s in ((0, 2048, (64, 32)), (2048, 3072, (16, 64)), (3072, 5120, (64, 32)), (5120, 9216, (64, 64)), (9216, 10240, (16, 64))))
    h = lambda a: a.astype(np.float32).astype(np.float16).astype(np.float64)  # noqa: E731
    def mm(W, x):  # half accumulator fragments, m16n16k16
        acc = np.zeros((W.shape[0], x.shape[1]))
        for k0 in range(0, W.shape[1], 16):
            acc = h(acc + W[:, k0:k0 + 16] @ x[k0:k0 + 16])
        return acc

    h1 = h(np.maximum(mm(W1, enc), 0))
    dens = h(mm(W2, h1))
    d = coords[:, 4:].astype(np.float32) * np.float32(2.0) - np.float32(1.0)
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    sh = np.stack([
        np.full_like(x, 0.28209479177387814), -0.48860251190291987 * y, 0.48860251190291987 * z, -0.48860251190291987 * x,
        1.0925484305920792 * x * y, -1.0925484305920792 * y * z, 0.94617469575755997 * z * z - 0.31539156525251999, -1.0925484305920792 * x * z,
        0.54627421529603959 * x * x - 0.54627421529603959 * y * y, 0.59004358992664352 * y * (-3.0 * x * x + y * y), 2.8906114426405538 * x * y * z,
        0.45704579946446572 * y * (1.0 - 5.0 * z * z), 0.3731763325901154 * z * (5.0 * z * z - 3.0), 0.45704579946446572 * x * (1.0 - 5.0 * z * z),
        1.4453057213202769 * z * (x * x - y * y), 0.59004358992664352 * x * (-x * x + 3.0 * y * y)]).astype(np.float32)
    rin = np.concatenate([dens, sh.astype(np.float16).astype(np.float64)], 0)
    out = h(mm(W5, h(np.maximum(mm(W4, h(np.maximum(mm(W3, rin), 0))), 0))))
    got = oracle.inference(coords).view(np.float16).astype(np.float64)
    gd = oracle.inference(coords, density_only=True).view(np.float16).astype(np.float64)
    assert np.abs(gd - dens).max() <= 1e-2 * np.abs(dens).max()  # float32-vs-double SH/accumulate noise flips an fp16 ulp at most
    assert np.allclose(got[3], dens[0])  # row 3 = density MLP out[0] (extract_density)
    assert np.abs(got[:3] - out[:3]).max() < 2e-2
    exact = (gd.astype(np.float16).view(np.uint16) == dens.astype(np.float16).view(np.uint16)).mean()
    assert exact > 0.99


def test_march_invariants(scene, oracle):
    model, occ = scene
    f = syn.make_frame(model, syn.fox_camera0(), 64, 36)
    pix = np.arange(0, 64 * 36, 7, dtype=np.uint32)
    rec, idx, cnt = oracle.march_trace(f, pix, 128)
    bits = np.unpackbits(occ, bitorder="little")
    min_step = np.float32(1.73205080757) / np.float32(1024)
    assert cnt.max() > 10
    for i in range(pix.size):
        n = min(int(cnt[i]), 128)
        t, dt = rec[i, :n, 0], rec[i, :n, 1]
        assert (np.diff(t) > 0).all()                                     # strictly advancing
        assert (dt >= min_step).all() and (dt <= min_step * 128).all()     # clamp of calc_dt
        assert np.allclose(dt, np.clip(t / 256.0, min_step, min_step * 128), rtol=1e-6)
        mip, cell = idx[i, :n, 0].astype(np.int64), idx[i, :n, 1].astype(np.int64)
        assert bits[mip * 128 ** 3 + cell].all()                            # every emitted sample sits in an occupied cell
        pos = rec[i, :n, 2:5]
        assert ((pos >= model.aabb_min) & (pos <= model.aabb_max)).all()
        # consecutive samples inside one occupied run are exactly dt apart (same dt lattice as skipped space)
        gaps = np.diff(t)
        assert (gaps >= dt[:-1] - 1e-6).all()


def test_render_empty_and_full_occupancy(scene):
    """Edge cases: empty occupancy -> nothing rendered, depth = 1e10; no bitfield -> every step sampled."""
    model, occ = scene
    f = syn.make_frame(model, syn.orbit_cameras(8)[2], 16, 9)
    o_empty = orc.Oracle(model.desc, model.params, np.zeros_like(occ))
    fb, depth, st, _ = o_empty.render(f)
    assert st.n_samples == 0 and st.n_hit == 0 and (fb == 0).all() and (depth == 1e10).all()
    o_none = orc.Oracle(model.desc, model.params, None)
    fb2, depth2, st2, _ = o_none.render(f)
    assert st2.n_samples > 16 * 9 * 50  # free space is sampled too without an occupancy grid
    assert np.isfinite(fb2).all()


def test_background_overblend(scene, oracle):
    model, _ = scene
    f = syn.make_frame(model, syn.orbit_cameras(8)[1], 32, 18)
    fb0, _, _, _ = oracle.render(f)
    bg = np.zeros((18, 32, 4), np.float32)
    bg[..., 1] = 0.5
    bg[..., 3] = 1.0
    fb1, _, _, _ = oracle.render(f, background=bg)
    a = fb0[..., 3:4]
    assert np.allclose(fb1, fb0 + bg * (1 - a), atol=1e-6)  # shade_kernel_nerf :2479
