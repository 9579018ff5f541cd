"""PNG writer, mosaic extent and the file names of the slice exports — no GPU needed (a stand-in renderer returns fixed pixels)."""
import os

import numpy as np
import pytest

from png_decode import decode_png
from nerfshop_b200 import mesh, slices


@pytest.mark.parametrize("channels,shape", [(1, (7, 13)), (1, (1, 1)), (4, (5, 9, 4)), (4, (3, 1, 4))])
def test_write_png_decodes_to_the_given_bytes(tmp_path, channels, shape):
    px = np.random.default_rng(sum(shape)).integers(0, 256, shape, dtype=np.uint8)
    p = str(tmp_path / "a.png")
    slices.write_png(p, px, channels)
    data = open(p, "rb").read()
    np.testing.assert_array_equal(decode_png(data), px)
    try:
        from PIL import Image
    except ImportError:
        return
    with Image.open(p) as im:
        assert im.mode == ("L" if channels == 1 else "RGBA")
        np.testing.assert_array_equal(np.asarray(im), px)


def test_write_png_rejects_a_shape_that_is_not_the_channel_count(tmp_path):
    with pytest.raises(ValueError):
        slices.write_png(str(tmp_path / "a.png"), np.zeros((4, 4, 3), np.uint8), 4)
    with pytest.raises(ValueError):
        slices.write_png(str(tmp_path / "a.png"), np.zeros((4, 4), np.uint8), 3)


def _reference_extent(res, swap):
    """save_density_grid_to_png's arithmetic (marching_cubes.cu:938-945): ndown = uint32_t(sqrtf(res_z')) in float32."""
    rx, ry, rz = (res[0], res[2], res[1]) if swap else tuple(res)
    ndown = int(np.sqrt(np.float32(rz)))
    nacross = (rz + ndown - 1) // ndown
    return rx * nacross, ry * ndown


def test_density_png_extent_equals_the_reference_for_every_slice_count(built_lib):
    for k in range(1, 2049):
        for res, swap in (((5, 7, k), False), ((5, 7, k), True), ((5, k, 7), True)):
            assert slices.density_png_extent(res, swap) == _reference_extent(res, swap), (res, swap)


def test_density_png_extent_rejects_empty_grids(built_lib):
    from nerfshop_b200 import abi

    for res in ((0, 4, 4), (4, -1, 4), (4, 4, 0)):
        with pytest.raises(abi.NsbError):
            slices.density_png_extent(res)


class _Host:
    """Stands in for a CUDA tensor: .cpu().numpy() / .cpu().tolist()."""

    def __init__(self, a):
        self.a = np.asarray(a)

    def cpu(self):
        return self

    def numpy(self):
        return self.a

    def tolist(self):
        return self.a.tolist()


class _FakeRenderer:
    """Records the calls slices.py makes and answers with pixels of the shapes the device returns."""

    def __init__(self):
        self.calls = []

    def density_on_grid(self, res3d, aabb, train_aabb):
        self.calls.append(("density_on_grid", tuple(int(v) for v in res3d)))
        return "grid"

    def density_png(self, density, res3d, thresh, density_range, swap_y_z):
        self.calls.append(("density_png", tuple(int(v) for v in res3d), thresh, density_range, swap_y_z))
        w, h = slices.density_png_extent(res3d, swap_y_z)
        return _Host(np.arange(w * h, dtype=np.uint32).astype(np.uint8).reshape(h, w)), _Host([11, 22])

    def rgba_on_grid(self, res3d, aabb, train_aabb, ray_dir, rgb_activation, density_activation):
        self.calls.append(("rgba_on_grid", tuple(int(v) for v in res3d), tuple(ray_dir)))
        return "rgba"

    def rgba_png(self, rgba, res3d, swap_y_z):
        rx, ry, rz = (int(v) for v in res3d)
        h, n = (rz, ry) if swap_y_z else (ry, rz)
        return _Host(np.arange(n * h * rx * 4, dtype=np.uint32).astype(np.uint8).reshape(n, h, rx, 4))


BOX = ((-1.3, -1.1, -0.9), (2.2, 2.1, 2.4))  # not a cube: 3.5 x 3.2 x 3.3


@pytest.mark.parametrize("flip", [False, True])
def test_density_slices_file_name_and_res3d_are_the_references(built_lib, tmp_path, flip):
    r = _FakeRenderer()
    res3d, counts = slices.compute_and_save_png_slices(r, str(tmp_path / "scene"), 100, BOX, BOX, thresh=1.5, density_range=2.0, flip_y_and_z_axes=flip)
    want = mesh.get_marching_cubes_res(100, BOX)
    np.testing.assert_array_equal(res3d, want)
    assert list(want) == [112, 96, 96]  # get_marching_cubes_res(100, BOX): round(diag * 100 / 3.5), up to multiples of 16
    # snprintf(".density_slices_%dx%dx%d.png", res3d) with res3d before the swap (testbed.cu:361-364)
    assert os.listdir(tmp_path) == ["scene.density_slices_112x96x96.png"]
    assert counts == (11, 22)
    assert r.calls[1] == ("density_png", (112, 96, 96), 1.5, 2.0, flip)
    img = decode_png(open(tmp_path / "scene.density_slices_112x96x96.png", "rb").read())
    assert img.shape[::-1] == slices.density_png_extent(want, flip)


@pytest.mark.parametrize("flip", [False, True])
def test_rgba_sequence_file_names_and_view_direction_are_the_references(built_lib, tmp_path, flip):
    r = _FakeRenderer()
    box = ((0, 0, 0), (1.0, 0.5, 0.3))
    names = slices.compute_and_save_rgba_png_sequence(r, str(tmp_path), 100, box, box, flip_y_and_z_axes=flip)
    assert r.calls == [("rgba_on_grid", (112, 64, 32), (0.0, 1.0, 0.0) if flip else (0.0, 0.0, 1.0))]  # testbed.cu:959
    w, h, n = (112, 32, 64) if flip else (112, 64, 32)  # after the swap: rows of res_x, res_z rows, res_y slices
    assert sorted(os.listdir(tmp_path / "rgba_slices")) == ["%04d_%dx%d.png" % (z, w, h) for z in range(n)]
    assert names == [str(tmp_path / "rgba_slices" / ("%04d_%dx%d.png" % (z, w, h))) for z in range(n)]
    img = decode_png(open(names[3], "rb").read())
    np.testing.assert_array_equal(img, np.arange(n * h * w * 4, dtype=np.uint32).astype(np.uint8).reshape(n, h, w, 4)[3])
