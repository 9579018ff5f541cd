"""Mesh extraction: the reference's marching-cubes entry points on top of the C ABI (nsb_density_on_grid, nsb_marching_cubes,
nsb_mesh_shade, nsb_mesh_download).

  get_marching_cubes_res        <- get_marching_cubes_res (marching_cubes.cu:48-55)
  compute_marching_cubes_mesh   <- Testbed::compute_marching_cubes_mesh (python_api.cu:105-126) over Testbed::marching_cubes
  save_mesh                     <- save_mesh (marching_cubes.cu:760-896)
  compute_and_save_marching_cubes_mesh <- Testbed::compute_and_save_marching_cubes_mesh (testbed.cu:337-343)
  optimise_mesh_step            <- Testbed::optimise_mesh_step (testbed_nerf.cu:4470-4513), the GUI's "Optimize mesh"

Arrays have the reference's row count: n_vertices rounded up to 128 (marching_cubes.cu:751-753). The padding rows sit at the
origin, carry the network's colour there and a zero normal.
"""
from __future__ import annotations

import os

import numpy as np

from . import abi


def get_marching_cubes_res(res_1d: int, aabb) -> np.ndarray:
    """The per-axis resolution for a longest-axis resolution res_1d, each rounded up to a multiple of 16 (float32 like the reference)."""
    mn, mx = np.asarray(aabb[0], np.float32), np.asarray(aabb[1], np.float32)
    diag = mx - mn
    scale = np.float32(res_1d) / diag.max()
    res = (diag * scale + np.float32(0.5)).astype(np.int32)
    return ((res.astype(np.int64) + 15) // 16 * 16).astype(np.int32)


def _normalized(v: np.ndarray) -> np.ndarray:
    """Eigen's normalized() per row in float32: x*x + (y*y + z*z), divided by its square root; zero rows stay zero."""
    v = np.asarray(v, np.float32)
    n2 = v[:, 0] * v[:, 0] + (v[:, 1] * v[:, 1] + v[:, 2] * v[:, 2])
    out = v.copy()
    ok = n2 > 0
    out[ok] = v[ok] / np.sqrt(n2[ok])[:, None]
    return out


def compute_marching_cubes_mesh(renderer, res3d, aabb, thresh: float, train_aabb, rgb_activation: int = abi.NSB_ACT_LOGISTIC,
                                linear_colors: bool = False) -> dict:
    """{V, N, C, F} of the field's iso-surface at `thresh` over `aabb` (res3d rounded up to multiples of 16, testbed_nerf.cu:4615-4617).
    N is normalised, as python_api.cu:119-122 does on the host; F is int32 [n_triangles, 3]. The renderer needs a model and a running
    density grid (nsb_upload_density_grid or nsb_update_density_grid)."""
    res = [((int(r) + 15) // 16) * 16 for r in res3d]
    density = renderer.density_on_grid(res, aabb, train_aabb)
    nv, ni = renderer.marching_cubes(density, res, aabb, thresh)
    renderer.mesh_shade(train_aabb, rgb_activation, linear_colors)
    m = renderer.mesh_download(nv, ni)
    return dict(V=m["V"], N=_normalized(m["N"]), C=m["C"], F=m["F"].astype(np.int32))


def save_mesh(path: str, mesh: dict, nerf_scale: float, nerf_offset, unwrap_it: bool = False) -> None:
    """Writes mesh (V, N, C, F) to `path`: PLY when its extension is `ply`, OBJ otherwise, in the reference's text format, each face
    written in reversed vertex order. Positions are (V - offset) / scale. N is normalised here, as the reference does: pass the normals
    as the device stores them (NerfRenderer.mesh_download), which is what compute_and_save_marching_cubes_mesh writes; normalising the
    already normalised N of compute_marching_cubes_mesh can change a last bit."""
    if unwrap_it:
        raise NotImplementedError("save_mesh: the UV unwrap (unwrap_it) is not implemented")
    V = np.asarray(mesh["V"], np.float32)
    N = _normalized(mesh["N"])
    Cc = np.asarray(mesh["C"], np.float32)
    F = np.asarray(mesh["F"]).reshape(-1).astype(np.uint32)
    P = (V - np.asarray(nerf_offset, np.float32)) / np.float32(nerf_scale)
    out = []
    ext = os.path.basename(path).rpartition(".")
    if ext[1] and ext[2] == "ply":
        c8 = np.clip(Cc * np.float32(255.0), np.float32(0.0), np.float32(255.0)).astype(np.uint8)
        out.append("ply\nformat ascii 1.0\ncomment output from https://github.com/NVlabs/instant-ngp\n"
                   f"element vertex {V.shape[0]}\nproperty float x\nproperty float y\nproperty float z\nproperty float nx\nproperty float ny\n"
                   f"property float nz\nproperty uchar red\nproperty uchar green\nproperty uchar blue\nelement face {F.size // 3}\n"
                   "property list uchar int vertex_index\nend_header\n")
        for p, n, c in zip(P.tolist(), N.tolist(), c8.tolist()):
            out.append("%0.5f %0.5f %0.5f %0.3f %0.3f %0.3f %d %d %d\n" % (p[0], p[1], p[2], n[0], n[1], n[2], c[0], c[1], c[2]))
        for i in range(0, F.size, 3):
            out.append("3 %d %d %d\n" % (F[i + 2], F[i + 1], F[i]))
    else:
        cc = np.clip(Cc, np.float32(0.0), np.float32(1.0))
        for p, c in zip(P.tolist(), cc.tolist()):
            out.append("v %0.5f %0.5f %0.5f %0.3f %0.3f %0.3f\n" % (p[0], p[1], p[2], c[0], c[1], c[2]))
        for n in N.tolist():
            out.append("vn %0.5f %0.5f %0.5f\n" % (n[0], n[1], n[2]))
        for i in range(0, F.size, 3):
            a, b, c = int(F[i + 2]) + 1, int(F[i + 1]) + 1, int(F[i]) + 1
            out.append(f"f {a}//{a} {b}//{b} {c}//{c}\n")
    with open(path, "w", newline="\n") as fh:
        fh.write("".join(out))


def compute_and_save_marching_cubes_mesh(renderer, path: str, res3d, aabb, thresh: float, train_aabb, nerf_scale: float, nerf_offset,
                                         rgb_activation: int = abi.NSB_ACT_LOGISTIC, linear_colors: bool = False) -> None:
    """Meshes like compute_marching_cubes_mesh and writes the file from the device's unnormalised normals, as the reference does."""
    res = [((int(r) + 15) // 16) * 16 for r in res3d]
    density = renderer.density_on_grid(res, aabb, train_aabb)
    nv, ni = renderer.marching_cubes(density, res, aabb, thresh)
    renderer.mesh_shade(train_aabb, rgb_activation, linear_colors)
    save_mesh(path, renderer.mesh_download(nv, ni), nerf_scale, nerf_offset)


def optimise_mesh_step(renderer, n_steps: int, thresh: float, train_aabb, smooth_amount: float = 2048.0, density_amount: float = 128.0,
                       inflate_amount: float = 1.0) -> None:
    """Moves the renderer's current mesh (the last marching_cubes) towards the `thresh` iso-surface of the raw density while smoothing it:
    n_steps Adam steps on every vertex row, padding rows included. The defaults are the reference's (marching_cubes.h:32-34). Read the result
    with renderer.mesh_download: the normals are those of the positions before the last step; the colours are not recomputed."""
    renderer.mesh_optimise(n_steps, thresh, train_aabb, smooth_amount, density_amount, inflate_amount)
