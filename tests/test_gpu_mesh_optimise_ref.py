"""nsb_mesh_optimise against the reference's own optimisation gradient (oracle/_ref/libnerfshop_ref_mesh_opt_cuda.so: compute_mesh_1ring and
compute_mesh_opt_gradients of marching_cubes.cu compiled by nvcc), through tests/ref_golden.py: where that build is absent the stored results
replay.

tiny-cuda-nn is absent, so nsb_density_gradient stands in for NerfNetwork::density + input_gradient(3) (its output goes to the reference in
the reference's layout: rows of 7 floats, the gradient in the first 3) and the restated tcnn Adam (oracle/mesh_opt_oracle.cpp) runs after the
reference's gradient. One step's positions are compared with nsb_mesh_optimise's.

The reference's 1-ring sums and normals are float atomics, so on a vertex whose triangles land in another order its sums can differ in the
last bits. Where the reference's sums and normals equal this repository's (ascending triangle order) bit for bit, the opt gradient and the
moved position must be bit-identical. Elsewhere the opt gradient differs by rounding only, and Adam's first step moves a coordinate by
lr * m / (sqrt(v) + eps), whose size is lr to within a few ulps whatever the gradient's magnitude: the new position may differ by one
rounding of the new position plus a few ulps of the step (which show where the position is near 0), and only a gradient component that
changes sign could move it further. Measured on the H100: 42 % of the rows agree bit for bit; of the rest, 5 coordinates differ, by at most 2 ulp.
"""
import numpy as np
import pytest

import ref_golden as rg
from oracle import ref_mesh_opt, ref_mesh_opt_build

HAVE = ref_mesh_opt_build.build() is not None
pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not (HAVE or rg._stored("test_gpu_mesh_optimise_ref")),
                                                  reason="neither oracle/_ref nor stored reference results (tests/golden/ref/)")]

AABB = ((-1.5, -1.5, -1.5), (2.5, 2.5, 2.5))
RES = 64
K = (2048.0, 128.0, 1.0)  # smooth, density, inflate: the reference's defaults (marching_cubes.h:32-34)


@pytest.fixture(scope="module")
def mr(scene, built_lib):
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


def _rows(theirs, n):
    """The rows a stored (sampled) reference result keeps, all rows for a live one."""
    return np.asarray(theirs.rows) if isinstance(theirs, rg.Sampled) else np.arange(n)


def test_one_step_vs_reference(mr):
    from oracle import mesh_opt_oracle as mo

    d = mr.density_on_grid((RES, RES, RES), AABB, AABB)
    v = d.cpu().numpy().reshape(-1)
    t = float(np.median(v[v > -10000.0]))
    nv, ni = mr.marching_cubes(d, (RES, RES, RES), AABB, t)
    m0 = mr.mesh_download(nv, ni, shaded=False)
    V0, F = m0["V"], m0["F"]
    coords = np.zeros((V0.shape[0], 7), np.float32)
    coords[:, :3] = (V0 - np.float32(-1.5)) / np.float32(4.0)  # warp_position; exact for this power-of-two box
    coords[:, 4:] = 0.5
    grad, dens = mr.density_gradient(coords)
    g7 = np.zeros((V0.shape[0], 7), np.float32)  # the reference reads the gradient in place of its network inputs (stride 7)
    g7[:, :3] = grad
    g_ref, s_ref, n_ref = rg._call(HAVE, ref_mesh_opt.opt_gradients if HAVE else None, V0, F, dens, g7, t, *K)
    rows = _rows(g_ref, V0.shape[0])
    g_ref, s_ref, n_ref = (np.asarray(a).view(np.ndarray) for a in (g_ref, s_ref, n_ref))
    s_our, n_our, g_our = (a[rows] for a in mo.mesh_opt_gradient(V0, F, dens, grad, t, *K))

    mr.mesh_optimise(1, t, AABB)
    V1 = mr.mesh_download(nv, ni, shaded=False)["V"][rows]
    P_ref, _ = mo.adam_step(V0[rows], g_ref)
    V0r = V0[rows]

    agree_with_reference(rows, nv, V1, P_ref, g_our, g_ref, s_our, s_ref, n_our, n_ref, min_agree=0.3)
    # the step moved the mesh as the reference's would: by about lr per coordinate with a non-zero gradient
    moved = np.abs(V1 - V0r)
    assert (moved <= 1.01e-4).all() and (moved > 0).mean() > 0.9


def agree_with_reference(rows, nv, V1, P_ref, g_our, g_ref, s_our, s_ref, n_our, n_ref, min_agree):
    """The agreement rule on the compared rows: bit for bit where the reference's atomic 1-ring sums and normals equal this repository's
    (and on the padding rows, which have no triangles), the documented tolerance elsewhere. Returns the share of rows whose sums agree."""
    agree = (s_ref.view(np.uint32) == s_our.view(np.uint32)).all(1) & (n_ref.view(np.uint32) == n_our.view(np.uint32)).all(1)
    padding = rows >= nv
    print(f"\n{rows.size} rows compared ({nv} vertices): 1-ring sums and normals bit-equal on {100 * agree.mean():.2f} %; "
          f"positions bit-equal on {100 * (V1 == P_ref).all(1).mean():.2f} %")
    # the atomics reorder the sums of most vertices with more than a few triangles (measured: 42 % of the rows agree bit for bit); the
    # bit-exact check below covers those rows and the padding, which have no triangles
    assert agree.mean() > min_agree and agree[padding].all()
    # where the atomic sums agree: the reference's opt gradient and the moved positions, bit for bit (padding rows included)
    np.testing.assert_array_equal(g_our[agree].view(np.uint32), g_ref[agree].view(np.uint32))
    np.testing.assert_array_equal(V1[agree].view(np.uint32), P_ref[agree].view(np.uint32))
    # elsewhere: the gradient differs by the summation order only, the position by at most one rounding where its sign is the same
    rest = ~agree
    rel = np.abs(g_our[rest] - g_ref[rest]) / np.maximum(np.abs(g_ref[rest]), 1e-30)
    same_sign = np.sign(g_our[rest]) == np.sign(g_ref[rest])
    print(f"rows whose sums differ: {rest.sum()}; opt gradient relative difference max {rel[same_sign].max() if same_sign.any() else 0:.2e}; "
          f"coordinates with a sign change: {(~same_sign).sum()}")
    assert (~same_sign).sum() <= max(2, int(1e-3 * same_sign.size))
    # one rounding of the new position, plus a few ulps of the step lr * m / (sqrt(v) + eps) itself, which show where the position is near 0,
    # plus the change of that first step, lr * g / (|g| + 10 eps), with the gradient: lr * 10 eps * |dg| / (|g| + 10 eps)^2, which only matters
    # where |g| is near 10 eps = 1e-7 (a smoothing gradient that nearly cancels)
    g_min = np.minimum(np.abs(g_our[rest]), np.abs(g_ref[rest])).astype(np.float64)
    dstep = 1.01e-4 * 1e-7 * np.abs(g_our[rest].astype(np.float64) - g_ref[rest]) / (g_min + 1e-7) ** 2
    tol = np.spacing(np.maximum(np.abs(V1[rest]), np.abs(P_ref[rest])).astype(np.float32)) + 4 * np.spacing(np.float32(1e-4)) + dstep
    off = np.abs(V1[rest] - P_ref[rest])
    print(f"positions that differ: {(off > 0).sum()} coordinates, at most {(off / tol)[same_sign].max() if same_sign.any() else 0:.2f} of the tolerance")
    assert (off[same_sign] <= tol[same_sign]).all()
    return agree.mean()
