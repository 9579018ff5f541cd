"""Times the mesh-extraction steps of Testbed::marching_cubes on the synthetic fox-config scene over its render AABB, with CUDA events:
nsb_density_on_grid at 256^3 and 512^3, nsb_marching_cubes (including its one count synchronisation) and nsb_mesh_shade, plus the device memory the
extraction holds (the context's buffers only grow, so this is also its peak), and the reference's marching_cubes_gpu on the same grid. The card, its power limit and SM clock are read in the same run.
  python tools/profile_mesh.py"""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from nerfshop_b200 import synthetic as syn  # noqa: E402
from nerfshop_b200.renderer import NerfRenderer  # noqa: E402
from oracle import ref_mesh, ref_mesh_build  # noqa: E402

AABB = ((-1.5, -1.5, -1.5), (2.5, 2.5, 2.5))
print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
model = syn.make_model(seed=1337)
occ = syn.make_occupancy(model)
r = NerfRenderer(0)
r.upload_model(model.desc, model.params)
r.upload_density_grid(np.unpackbits(occ, bitorder="little").astype(np.float32))


def timed(fn, reps):
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms[1:])), out


for res in (256, 512):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    free0 = torch.cuda.mem_get_info()[0]
    out = torch.empty(res ** 3, dtype=torch.float32, device="cuda")
    t_d, _ = timed(lambda: r.density_on_grid((res, res, res), AABB, AABB, out=out), 6)
    v = out.cpu().numpy()
    thresh = float(np.median(v[v > -10000.0]))
    t_mc, (nv, ni) = timed(lambda: r.marching_cubes(out, (res, res, res), AABB, thresh), 6)
    t_sh, _ = timed(lambda: r.mesh_shade(AABB), 6)
    free1 = torch.cuda.mem_get_info()[0]
    print(f"{res}^3: density_on_grid {t_d:.3f} ms = {res ** 3 / t_d / 1e6:.2f} Gsamples/s; marching_cubes {t_mc:.3f} ms "
          f"({nv} vertices, {ni // 3} triangles, thresh {thresh:.4f}); mesh_shade (normals + colours) {t_sh:.3f} ms; "
          f"device memory in use after the extraction: {(free0 - free1) / 2 ** 20:.1f} MiB beyond the start "
          f"(density grid {res ** 3 * 4 / 2 ** 20:.0f} MiB of it)", flush=True)
    ref = "not measured (oracle/_ref mesh build absent)"
    if ref_mesh_build.build() is not None:
        ms = [ref_mesh.marching_cubes(v, (res, res, res), AABB, thresh, want_ms=True)[2] for _ in range(4)]
        ref = f"{float(np.median(ms[1:])):.3f} ms"
    print(f"{res}^3: the reference's marching_cubes_gpu (oracle/_ref, nvcc sm_90a, same density and threshold): {ref}", flush=True)
    del out
r.close()
