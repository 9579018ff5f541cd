"""nsb_density_gradient on the H100 against the CPU restatement (oracle/mesh_opt_oracle.cpp), under both MLP accumulator policies:
the raw density is nsb_density's bit for bit, dfeat (dL/dfeatures * 128) meets the MLP contract, and the grid backward of the device's own
dfeat is the oracle's bit for bit. Ragged n (not a multiple of 128) and positions on lattice points of the grid levels."""
import ctypes as C

import numpy as np
import pytest

from conftest import random_coords

pytestmark = pytest.mark.gpu

POLICIES = {"f32": (0, 0), "f16": (1, 1)}  # device policy (NSB_MLP_ACC_*), oracle policy


@pytest.fixture(scope="module")
def gr(scene, built_lib):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nerfshop_b200.renderer import NerfRenderer

    model, _ = scene
    r = NerfRenderer(0)
    r.upload_model(model.desc, model.params)
    yield r
    r.close()


def _lattice_coords(model, n_per_level=16, seed=9):
    """Positions x with fma(scale_l, x, 0.5) an integer on one axis for some level l: the interpolation weight there is exactly 0."""
    from oracle import oracle as orc

    nl = model.desc.n_levels
    scale, res, off, size = np.zeros(nl, np.float32), np.zeros(nl, np.uint32), np.zeros(nl, np.uint32), np.zeros(nl, np.uint32)
    assert orc.lib().orc_level_table(C.byref(model.desc), *[a.ctypes.data_as(C.c_void_p) for a in (scale, res, off, size)]) == 0
    rng = np.random.default_rng(seed)
    rows = []
    for l in range(nl):
        s = np.float64(scale[l])
        for _ in range(n_per_level):
            c = random_coords(1, seed=int(rng.integers(1 << 30)))[0]
            k = int(rng.integers(1, max(2, int(s))))
            x = np.float32((k - 0.5) / s)
            for cand in (x, np.nextafter(x, np.float32(1)), np.nextafter(x, np.float32(0))):
                if float(np.float32(np.float64(s) * np.float64(cand) + 0.5)) == float(k):
                    c[int(rng.integers(3))] = cand
                    rows.append(c)
                    break
    return np.array(rows, np.float32)


def _coords(model):
    c = random_coords(5037, seed=21)
    c[:5, :3] = [[0, 0, 0], [1, 1, 1], [0.5, 0.5, 0.5], [0.25, 0.75, 0.125], [1, 0, 0.5]]
    lat = _lattice_coords(model)
    assert lat.shape[0] >= 64
    return np.concatenate([c, lat])


def _ulps(a, b):
    """fp16 ulp distance on the bit patterns, +0 and -0 counted equal."""
    ia = np.where(a & 0x8000, -(a & 0x7FFF).astype(np.int64), (a & 0x7FFF).astype(np.int64))
    ib = np.where(b & 0x8000, -(b & 0x7FFF).astype(np.int64), (b & 0x7FFF).astype(np.int64))
    return np.abs(ia - ib)


@pytest.mark.parametrize("policy", sorted(POLICIES))
def test_density_gradient_against_the_oracle(gr, scene, oracle, policy):
    from nerfshop_b200 import abi
    from oracle import mesh_opt_oracle as mo

    model, _ = scene
    dev_policy, orc_policy = POLICIES[policy]
    coords = _coords(model)
    n = coords.shape[0]
    assert n % 128 != 0
    gr.set_mlp_accumulator(dev_policy)
    old = mo.set_mlp_policy(orc_policy)
    try:
        grad, dens, dfeat = gr.density_gradient(coords, want_dfeat=True)
        raw = gr.density(coords)[0]
        g_o, df_o, dens_o = mo.density_gradient(oracle, coords)
        g_given, _, _ = mo.density_gradient(oracle, coords, dfeat=dfeat)
    finally:
        mo.set_mlp_policy(old)
        gr.set_mlp_accumulator(abi.NSB_MLP_ACC_F16)
    # the forward is nsb_density's, bit for bit
    np.testing.assert_array_equal(dens, raw)
    # dfeat meets the MLP contract against the oracle
    u = _ulps(dfeat, df_o)
    eq = (u == 0).mean()
    print(f"\n{policy}: dfeat {100 * eq:.3f} % bit-equal, max {u.max()} ulp, 99.99th pct {np.percentile(u, 99.99)}; density {100 * (dens == dens_o).mean():.3f} % bit-equal to the oracle")
    assert eq >= 0.999 and u.max() <= 4
    # the grid backward of the device's dfeat is the oracle's bit for bit
    np.testing.assert_array_equal(grad.view(np.uint32), g_given.view(np.uint32))
    assert np.isfinite(grad).all() and (np.abs(grad).max(1) > 0).mean() > 0.99


def test_in_place_stride_7_equals_separate_output(gr, scene):
    import torch

    model, _ = scene
    coords = _coords(model)
    n = coords.shape[0]
    n_pad = (n + 127) // 128 * 128
    grad, dens = gr.density_gradient(coords)
    c = torch.as_tensor(coords).cuda().contiguous()
    d = torch.zeros(n_pad, dtype=torch.int16, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    assert gr.lib.nsb_density_gradient(gr.ctx, c.data_ptr(), n, c.data_ptr(), 7, d.data_ptr(), None, n_pad, st) == 0
    torch.cuda.synchronize()
    out = c.cpu().numpy()
    np.testing.assert_array_equal(out[:, :3].view(np.uint32), grad.view(np.uint32))
    np.testing.assert_array_equal(out[:, 3:].view(np.uint32), coords[:, 3:].view(np.uint32))  # dt and dir untouched
    np.testing.assert_array_equal(d.cpu().numpy().view(np.uint16)[:n], dens)


def test_status_codes(scene, built_lib):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nerfshop_b200 import abi
    from nerfshop_b200.renderer import NerfRenderer

    model, _ = scene
    r = NerfRenderer(0)
    c = torch.zeros((128, 7), device="cuda")
    g = torch.zeros((128, 3), device="cuda")
    assert r.lib.nsb_density_gradient(r.ctx, c.data_ptr(), 128, g.data_ptr(), 3, None, None, 128, None) == abi.NSB_ERR_STATE  # no model
    r.upload_model(model.desc, model.params)
    assert r.lib.nsb_density_gradient(r.ctx, c.data_ptr(), 128, g.data_ptr(), 2, None, None, 128, None) == abi.NSB_ERR_INVALID
    assert r.lib.nsb_density_gradient(r.ctx, c.data_ptr(), 128, g.data_ptr(), 3, None, None, 64, None) == abi.NSB_ERR_INVALID
    assert r.lib.nsb_density_gradient(r.ctx, None, 128, g.data_ptr(), 3, None, None, 128, None) == abi.NSB_ERR_INVALID
    assert r.lib.nsb_density_gradient(r.ctx, c.data_ptr(), 128, g.data_ptr(), 3, None, None, 128, None) == abi.NSB_OK
    torch.cuda.synchronize()
    r.close()
