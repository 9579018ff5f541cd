"""Density and RGBA slices against the reference's own code (oracle/_ref/libnerfshop_ref_slices_cuda.so: the RGBA grid kernels of
testbed_nerf.cu compiled by nvcc, the PNG writers of marching_cubes.cu compiled as host code), through tests/ref_golden.py: where that
build is absent the stored results replay.

Scene: the synthetic fox-config model, train AABB [-1.5, 2.5]^3, the occupancy as the running density grid (0/1 floats). The box has
extents that are not powers of two and a 48-point axis; 32 slices make a 7 x 5 mosaic with 3 empty tiles. This repository's nsb_inference
stands in for tiny-cuda-nn's Network::inference between the reference's kernels (rows 0-3 of its fp16 output cast to float).
"""
import os

import numpy as np
import pytest

import ref_golden as rg
from png_decode import decode_png
from nerfshop_b200 import abi, slices
from oracle import ref_slices_build

HAVE = ref_slices_build.build() is not None
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not (HAVE or rg._stored("test_gpu_slices")),
                                                  reason="neither oracle/_ref nor stored reference results (tests/golden/ref/)")]

TRAIN = np.array([[-1.5, -1.5, -1.5], [2.5, 2.5, 2.5]], np.float32)
BOX = np.array([[-1.3, -1.1, -0.9], [2.2, 2.1, 2.4]], np.float32)
RES = np.array([48, 16, 32], np.int32)
OBLIQUE = np.array([0.48, -0.6, 0.64], np.float32)


@pytest.fixture(autouse=True)
def _device_for_the_live_reference():
    import torch

    if HAVE and not torch.cuda.is_available():
        pytest.skip("no CUDA device for the reference build")


def R(name, *args):
    from oracle import ref_slices

    return rg._call(HAVE, getattr(ref_slices, name) if HAVE else None, *args)


@pytest.fixture(scope="module")
def sr(scene, built_lib):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from nerfshop_b200.renderer import NerfRenderer

    model, occ = scene
    r = NerfRenderer(0)
    r.upload_model(model.desc, model.params)
    r.upload_density_grid(np.unpackbits(occ, bitorder="little").astype(np.float32))
    yield r
    r.close()


def _ref_rgba(sr, res, box, train, ray_dir, rgb_act, density_act):
    """get_rgba_on_grid's structure: the reference's positions, nsb_inference for Network::inference, the reference's compute_nerf_density."""
    from oracle import ref_slices

    coords = ref_slices.grid_coords(res, box, train, ray_dir)
    rgbd = sr.inference(coords[:, :7])[:4].view(np.float16).astype(np.float32).T
    return ref_slices.compute_nerf_density(rgbd, rgb_act, density_act)


RGBA_CASES = [((0.0, 0.0, 1.0), abi.NSB_ACT_LOGISTIC, abi.NSB_ACT_EXPONENTIAL),
              ((0.0, 1.0, 0.0), abi.NSB_ACT_LOGISTIC, abi.NSB_ACT_EXPONENTIAL),
              (tuple(OBLIQUE.tolist()), abi.NSB_ACT_LOGISTIC, abi.NSB_ACT_EXPONENTIAL),
              ((0.0, 0.0, 1.0), abi.NSB_ACT_EXPONENTIAL, abi.NSB_ACT_RELU)]


@pytest.mark.parametrize("policy", [abi.NSB_MLP_ACC_F16, abi.NSB_MLP_ACC_F32], ids=["f16", "f32"])
def test_rgba_on_grid_bit_exact_vs_reference(sr, policy):
    sr.set_mlp_accumulator(policy)
    res = np.array([48, 16, 16], np.int32)
    try:
        for ray_dir, ra, da in RGBA_CASES:
            d = np.array(ray_dir, np.float32)
            ours = sr.rgba_on_grid(res, BOX, TRAIN, d, ra, da).reshape(-1, 4)
            ref_rgba = rg._call(HAVE, (lambda *a: _ref_rgba(sr, *a)) if HAVE else None, res, BOX, TRAIN, d, ra, da)
            o, t = rg.ref.match(ours.cpu().numpy(), ref_rgba)
            assert o.shape[0] > 100
            a = o[:, 3]
            assert (a > 0).any() and (a < 1).any()  # both empty and dense points are checked
            np.testing.assert_array_equal(o.view(np.uint32), t.view(np.uint32))
    finally:
        sr.set_mlp_accumulator(abi.NSB_MLP_ACC_F16)  # the context's default


def _density(sr):
    import torch

    d = sr.density_on_grid(RES, BOX, TRAIN)
    torch.cuda.synchronize()
    dn = d.cpu().numpy().reshape(-1)
    assert (dn == -10000.0).any() and (dn > -10000.0).any()  # filtered cells are present
    return d, dn, float(np.median(dn[dn > -10000.0]))


@pytest.mark.parametrize("swap", [False, True])
def test_density_mosaic_and_counts_byte_identical_to_reference(sr, swap):
    d, dn, t = _density(sr)
    for rng in (4.0, 0.001):
        px, counts = sr.density_png(d, RES, t, rng, swap)
        px, counts = px.cpu().numpy(), counts.cpu().numpy()
        name, ref_px, ref_counts = R("density_png", dn, RES, t, swap, rng)
        assert name == "ref" and ref_px.shape == px.shape == slices.density_png_extent(RES, swap)[::-1]
        assert px.tobytes() == ref_px.tobytes()
        np.testing.assert_array_equal(counts, ref_counts)
        assert counts[0] > 0 and counts[1] > 0
        if rng < 0.01:
            assert (px == 255).any() and (px == 0).any()  # saturation both ways
    if not swap:  # 32 slices: ndown 5, nacross 7, the last 3 tiles are empty
        w, h = slices.density_png_extent(RES, False)
        assert (w, h) == (48 * 7, 16 * 5) and (px[4 * 16:, 4 * 48:] == 0).all()
    px2, counts2 = sr.density_png(d, RES, t, 4.0, swap)
    px1, counts1 = sr.density_png(d, RES, t, 4.0, swap)
    assert px1.cpu().numpy().tobytes() == px2.cpu().numpy().tobytes() and (counts1.cpu() == counts2.cpu()).all()


@pytest.mark.parametrize("swap", [False, True])
def test_rgba_slices_byte_identical_to_reference(sr, swap):
    rgba = sr.rgba_on_grid(RES, BOX, TRAIN, (0.0, 1.0, 0.0) if swap else (0.0, 0.0, 1.0))
    ours = sr.rgba_png(rgba, RES, swap).cpu().numpy()
    names, ref_px = R("rgba_png", rgba.cpu().numpy(), RES, swap)
    n, h, w = ours.shape[:3]
    assert names == ["%04d_%dx%d.png" % (z, w, h) for z in range(n)]
    assert ours.shape == ref_px.shape and ours.tobytes() == ref_px.tobytes()


def test_end_to_end_files_are_the_device_bytes_and_leave_the_context_as_it_was(sr, scene, tmp_path):
    import torch
    from nerfshop_b200 import mesh
    from nerfshop_b200 import synthetic as syn

    model, _ = scene
    frame = syn.make_frame(model, syn.orbit_cameras(120)[17], 128, 72)
    before = sr.render(frame)[0].clone()
    torch.cuda.synchronize()
    res3d = mesh.get_marching_cubes_res(48, BOX)
    files = []
    for run in range(2):
        out = tmp_path / str(run)
        out.mkdir()
        r3, counts = slices.compute_and_save_png_slices(sr, str(out / "scene"), 48, BOX, TRAIN, 1.0, 4.0, False)
        np.testing.assert_array_equal(r3, res3d)
        names = slices.compute_and_save_rgba_png_sequence(sr, str(out), 48, BOX, TRAIN, flip_y_and_z_axes=True)
        files.append([str(out / ("scene.density_slices_%dx%dx%d.png" % tuple(res3d)))] + names)
    assert [os.path.basename(f) for f in files[0]] == [os.path.basename(f) for f in files[1]]
    for a, b in zip(*files):
        assert open(a, "rb").read() == open(b, "rb").read()
    d = sr.density_on_grid(res3d, BOX, TRAIN)
    px, dev_counts = sr.density_png(d, res3d, 1.0, 4.0, False)
    assert decode_png(open(files[0][0], "rb").read()).tobytes() == px.cpu().numpy().tobytes()
    assert counts == tuple(dev_counts.cpu().tolist())
    rgba_px = sr.rgba_png(sr.rgba_on_grid(res3d, BOX, TRAIN, (0.0, 1.0, 0.0)), res3d, True).cpu().numpy()
    assert len(files[0]) - 1 == rgba_px.shape[0]
    for z, f in enumerate(files[0][1:]):
        assert decode_png(open(f, "rb").read()).tobytes() == rgba_px[z].tobytes()
    after = sr.render(frame)[0]
    torch.cuda.synchronize()
    assert torch.equal(before.view(torch.int32), after.view(torch.int32))


def test_validation(sr, scene, built_lib):
    import ctypes as C

    import torch
    from nerfshop_b200.renderer import NerfRenderer

    model, _ = scene
    lib = sr.lib
    dev = torch.device("cuda", sr.device)
    bare = NerfRenderer(0)
    try:
        with pytest.raises(abi.NsbError, match="status 3"):
            bare.rgba_on_grid(RES, BOX, TRAIN, (0, 0, 1))  # no model
        bare.upload_model(model.desc, model.params)
        with pytest.raises(abi.NsbError, match="status 3"):
            slices.compute_and_save_png_slices(bare, "/nonexistent/x", 48, BOX, TRAIN)  # no density grid: nsb_density_on_grid
    finally:
        bare.close()
    q = abi.NsbGridQuery()
    q.res[:] = [48, 16, 32]
    out = torch.empty(48 * 16 * 32 * 4, dtype=torch.float32, device=dev)
    d3 = (C.c_float * 3)(0, 0, 1)
    res = (C.c_int32 * 3)(48, 16, 32)
    px = torch.empty(48 * 16 * 32 * 4, dtype=torch.uint8, device=dev)
    cnt = torch.empty(2, dtype=torch.int64, device=dev)
    INVALID = abi.NSB_ERR_INVALID
    assert lib.nsb_rgba_on_grid(sr.ctx, None, d3, 2, 3, out.data_ptr(), None) == INVALID
    assert lib.nsb_rgba_on_grid(sr.ctx, C.byref(q), None, 2, 3, out.data_ptr(), None) == INVALID
    assert lib.nsb_rgba_on_grid(sr.ctx, C.byref(q), d3, 2, 3, None, None) == INVALID
    assert lib.nsb_rgba_on_grid(sr.ctx, C.byref(q), d3, 4, 3, out.data_ptr(), None) == INVALID
    assert lib.nsb_rgba_on_grid(sr.ctx, C.byref(q), d3, 2, -1, out.data_ptr(), None) == INVALID
    for bad in ([48, 17, 32], [0, 16, 32], [-16, 16, 32]):
        q.res[:] = bad
        assert lib.nsb_rgba_on_grid(sr.ctx, C.byref(q), d3, 2, 3, out.data_ptr(), None) == INVALID
    grid = out[: 48 * 16 * 32]
    assert lib.nsb_density_png(sr.ctx, None, res, 1.0, 4.0, 0, px.data_ptr(), cnt.data_ptr(), None) == INVALID
    assert lib.nsb_density_png(sr.ctx, grid.data_ptr(), res, 1.0, 4.0, 0, None, cnt.data_ptr(), None) == INVALID
    assert lib.nsb_density_png(sr.ctx, grid.data_ptr(), res, 1.0, 4.0, 0, px.data_ptr(), None, None) == INVALID
    for rng in (0.0, -1.0, float("nan"), float("inf")):
        assert lib.nsb_density_png(sr.ctx, grid.data_ptr(), res, 1.0, rng, 0, px.data_ptr(), cnt.data_ptr(), None) == INVALID
    for bad in ((0, 16, 32), (48, -1, 32), (1 << 16, 1 << 16, 2)):
        r3 = (C.c_int32 * 3)(*bad)
        assert lib.nsb_density_png(sr.ctx, grid.data_ptr(), r3, 1.0, 4.0, 0, px.data_ptr(), cnt.data_ptr(), None) == INVALID
        assert lib.nsb_rgba_png(sr.ctx, out.data_ptr(), r3, 0, px.data_ptr(), None) == INVALID
    assert lib.nsb_rgba_png(sr.ctx, None, res, 0, px.data_ptr(), None) == INVALID
    assert lib.nsb_rgba_png(sr.ctx, out.data_ptr(), res, 0, None, None) == INVALID
    assert lib.nsb_rgba_png(None, out.data_ptr(), res, 0, px.data_ptr(), None) == INVALID
    assert lib.nsb_density_png_extent(None, 0, C.byref(C.c_uint32()), C.byref(C.c_uint32())) == INVALID
    # a density grid of any positive size, not only multiples of 16
    odd = (C.c_int32 * 3)(5, 3, 7)
    assert lib.nsb_density_png(sr.ctx, grid.data_ptr(), odd, 1.0, 4.0, 1, px.data_ptr(), cnt.data_ptr(), None) == abi.NSB_OK
    torch.cuda.synchronize()
