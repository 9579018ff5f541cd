"""The float64 network reference (tests/network_reference.py) pinned without a GPU: its premises (lattice features are table entries,
every exact model's sums are exact in fp16, the exact models together reach every weight), the CPU oracle equal to it bit for bit on
every exact model under both accumulator policies, and the oracle inside its intervals on random models."""
import numpy as np
import pytest

import network_reference as nr
from nerfshop_b200 import synthetic as syn
from oracle import oracle as orc


@pytest.fixture(scope="module")
def models():
    return nr.exact_models()


@pytest.fixture(scope="module")
def rows():
    return nr.exact_rows(2048, seed=3)


def test_lattice_features_are_table_entries(models, rows):
    coords, k = rows
    params, ws, table, _, _ = models["int0"]
    enc = orc.Oracle(nr.desc(), params, None).encode(coords).T.view(np.float16).astype(np.float64)
    feat, _, _ = nr.exact_reference(ws, table, coords, k)
    assert np.array_equal(enc[: k.shape[0]], feat[: k.shape[0]])
    assert np.isnan(enc[k.shape[0]:]).all()  # NaN / inf positions: every feature NaN
    assert (k < 0).any() and (k > 16).any()  # rows outside the cube are among them


def test_exact_models_are_certified_and_cover_every_weight(models, rows):
    coords, k = rows
    sub = []
    for name, (params, ws, table, units, skip) in models.items():
        feat, d, rgb = nr.exact_reference(ws, table, coords, k)
        sh = nr.sh4_f32(coords[:, 4:])
        if units is not None:
            nr.certificate(ws, feat, sh, units, skip)
        elif name.startswith("sh"):  # the probes return the fp16 SH values themselves
            kk = int(name[2:])
            r = [x for x in range(16) if x != 3]
            np.testing.assert_array_equal(rgb[:, r], sh[:, [(x + 8 * (kk // 32)) % 16 for x in r]])
        if name.startswith("int") or name.startswith("sh"):
            sub.append((ws, feat[:1024], sh[:1024]) if name.startswith("sh") else (ws, feat, sh))
    cov = nr.coverage(sub)
    for l, c in enumerate(cov):
        want = np.ones_like(c)
        if l == 4:
            want[3] = False  # W5 row 3: nsb_inference row 3 is the density, no output shows it
        missing = np.argwhere(want & ~c)
        assert missing.size == 0, f"W{l + 1}: weights no exact model reaches: {missing[:8].tolist()}"


def test_range_models_reach_their_edges(models, rows):
    coords, k = rows
    _, ws, table, _, _ = models["subnormal"]
    _, d, rgb = nr.exact_reference(ws, table, coords, k)
    fin = np.isfinite(coords[:, :3]).all(1)
    for v in (d[fin], rgb[fin]):
        nz = np.abs(v[v != 0])
        assert nz.min() == 2.0 ** -24 and (nz < 2.0 ** -14).mean() > 0.5
    _, ws, table, _, _ = models["top"]
    _, d, rgb = nr.exact_reference(ws, table, coords, k)
    assert np.abs(rgb[fin]).max() >= 2.0 ** 14 and np.abs(d[fin]).max() >= 2.0 ** 14
    _, ws, table, _, _ = models["overflow"]
    feat, d, rgb = nr.exact_reference(ws, table, coords, k)
    hot = feat[:, nr.OVERFLOW_FEATURE] == 2
    assert 0.1 < hot.mean() < 0.4
    assert np.isnan(d[hot]).all() and np.isnan(rgb[hot, 3]).all()
    assert (rgb[hot][:, [0, 1, 2] + list(range(4, 16))] == 0).all()  # NaN into L3, ReLU -> 0
    assert np.isfinite(d[~hot & fin]).all()
    # non-finite positions: density 0, rgb = the network on a zero density input
    bad = ~fin
    assert (d[bad] == 0).all()
    _, ws, table, _, _ = models["sh5"]
    _, d, rgb = nr.exact_reference(ws, table, coords, k)
    sh = nr.sh4_f32(coords[bad, 4:])
    assert np.array_equal(rgb[bad][:, :3], sh[:, :3])  # probe 5 routes SH columns 0-2 to rgb rows 0-2


@pytest.mark.parametrize("policy", [0, 1])
def test_oracle_equals_the_reference_on_every_exact_model(models, rows, policy):
    coords, k = rows
    old = orc.set_mlp_policy(policy)
    try:
        for name, (params, ws, table, _, _) in models.items():
            o = orc.Oracle(nr.desc(), params, None)
            _, d, rgb = nr.exact_reference(ws, table, coords, k)
            got_d = o.inference(coords, density_only=True).T
            got = o.inference(coords).T
            bad_d, bad = nr.mismatch(got_d, d), nr.mismatch(got, rgb)
            assert not bad_d.any(), f"{name}: density rows {np.argwhere(bad_d)[:4].tolist()}"
            assert not bad.any(), f"{name}: inference rows {np.argwhere(bad)[:4].tolist()}"
    finally:
        orc.set_mlp_policy(old)


def interval_models():
    """name -> parameter block: the synthetic fox model and two wider-gain seeds of the fox geometry."""
    return {"fox": syn.make_model(seed=1337).params, "seed7_gain1.6": nr.random_model(7, 1.6), "seed8_gain2": nr.random_model(8, 2.0)}


@pytest.mark.parametrize("policy", [0, 1])
def test_oracle_inside_the_interval_reference(policy):
    desc = syn.model_desc()
    old = orc.set_mlp_policy(policy)
    total = 0
    try:
        for name, params in interval_models().items():
            coords = nr.random_rows(40_000, seed=11)
            o = orc.Oracle(desc, params, None)
            feat = o.encode(coords).T.view(np.float16).astype(np.float64)
            ws, _ = nr.unpack(params)
            lo, hi = nr.forward_interval(ws, feat, nr.sh4_f32(coords[:, 4:]), acc16=policy == 1)
            got = np.concatenate([o.inference(coords, density_only=True).T, o.inference(coords).T], 1)
            w = nr.width_ulps(lo, hi).max(0)
            print(f"\n{name} policy {policy}: interval width per output (fp16 ulps of its scale), max over rows: {np.ceil(w).astype(int).tolist()}")
            out = nr.outside(got, lo, hi)
            assert not out.any(), f"{name}: {out.sum()} outputs outside their interval, first {np.argwhere(out)[:4].tolist()}"
            assert w[:16].max() <= nr.WIDTH_CAP[0] and w[16:].max() <= nr.WIDTH_CAP[1]
            total += coords.shape[0]
    finally:
        orc.set_mlp_policy(old)
    assert total >= 100_000
