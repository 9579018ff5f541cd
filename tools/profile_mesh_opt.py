"""Times mesh optimisation on the synthetic fox-config scene over its render AABB, with CUDA events: one step of nsb_mesh_optimise
(Testbed::optimise_mesh_step) on the 256^3 mesh (density and gradient at every vertex row, then the 1-ring + Adam step), and
nsb_density_gradient alone in samples/s on 2^22 random NerfCoordinate rows, both accumulator policies. The card, its power limit and SM
clock are read in the same run.
  python tools/profile_mesh_opt.py"""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

from conftest import random_coords  # noqa: E402
from nerfshop_b200 import abi  # noqa: E402
from nerfshop_b200 import synthetic as syn  # noqa: E402
from nerfshop_b200.renderer import NerfRenderer  # noqa: E402

AABB = ((-1.5, -1.5, -1.5), (2.5, 2.5, 2.5))
print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
model = syn.make_model(seed=1337)
occ = syn.make_occupancy(model)
r = NerfRenderer(0)
r.upload_model(model.desc, model.params)
r.upload_density_grid(np.unpackbits(occ, bitorder="little").astype(np.float32))


def timed(fn, reps, inner=1):
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(inner):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1) / inner)
    return float(np.median(ms))


res = 256
d = r.density_on_grid((res, res, res), AABB, AABB)
v = d.cpu().numpy()
thresh = float(np.median(v[v > -10000.0]))
nv, ni = r.marching_cubes(d, (res, res, res), AABB, thresh)
rows = (nv + 127) // 128 * 128
n = 1 << 22
c = torch.as_tensor(random_coords(n, seed=1)).cuda().contiguous()
g = torch.empty((n, 3), dtype=torch.float32, device="cuda")
out = torch.empty((16, n), dtype=torch.int16, device="cuda")
st = torch.cuda.current_stream().cuda_stream
for name, policy in (("fp16 accumulators", abi.NSB_MLP_ACC_F16), ("fp32 accumulators", abi.NSB_MLP_ACC_F32)):
    r.set_mlp_accumulator(policy)
    t_step = timed(lambda: r.mesh_optimise(1, thresh, AABB), 5, 10)
    t_grad = timed(lambda: abi.check(r.lib, r.lib.nsb_density_gradient(r.ctx, c.data_ptr(), n, g.data_ptr(), 3, None, None, n, st), "nsb_density_gradient"), 5, 10)
    t_dens = timed(lambda: abi.check(r.lib, r.lib.nsb_density(r.ctx, c.data_ptr(), n, out.data_ptr(), n, st), "nsb_density"), 5, 10)
    print(f"{name}: nsb_mesh_optimise 1 step on the {res}^3 mesh ({nv} vertices, {rows} rows, {ni // 3} triangles): {t_step:.3f} ms; "
          f"nsb_density_gradient on {n} rows: {t_grad:.3f} ms = {n / t_grad / 1e6:.3f} Gsamples/s "
          f"(nsb_density alone: {t_dens:.3f} ms = {n / t_dens / 1e6:.3f} Gsamples/s)", flush=True)
r.set_mlp_accumulator(abi.NSB_MLP_ACC_F16)
r.close()
