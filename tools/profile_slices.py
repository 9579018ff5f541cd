"""Times the slice exports on the synthetic fox-config scene over its render AABB at 256^3 and 512^3 under both MLP accumulator policies, with
CUDA events: nsb_rgba_on_grid, nsb_density_png, nsb_rgba_png, the device-to-host copy of the pixels and the host PNG encoding
(nerfshop_b200.slices.write_png, wall clock). Beside them, the reference's structure of get_rgba_on_grid: its position kernel
(generate_grid_samples_nerf_uniform_dir), nsb_inference in 1M-point batches standing in for Network::inference (plus the cast of rows 0-3
to float4), and compute_nerf_density, each from oracle/_ref. The card, its power limit and SM clock are read in the same run.
  python tools/profile_slices.py"""
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from nerfshop_b200 import abi, slices  # noqa: E402
from nerfshop_b200 import synthetic as syn  # noqa: E402
from nerfshop_b200.renderer import NerfRenderer  # noqa: E402
from oracle import ref_slices_build  # noqa: E402

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


def wall(fn, reps):
    s = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        s.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(s[1:]))


have_ref = ref_slices_build.build() is not None
if have_ref:
    from oracle import ref_slices
for res in (256, 512):
    n = res ** 3
    R3 = (res, res, res)
    rgba = torch.empty((n, 4), dtype=torch.float32, device="cuda")
    density = r.density_on_grid(R3, AABB, AABB)
    torch.cuda.synchronize()
    dn = density.reshape(-1)
    thresh = float(dn[dn > -10000.0].median())
    for policy, name in ((abi.NSB_MLP_ACC_F16, "f16"), (abi.NSB_MLP_ACC_F32, "f32")):
        r.set_mlp_accumulator(policy)
        t_rgba, _ = timed(lambda: r.rgba_on_grid(R3, AABB, AABB, (0.0, 0.0, 1.0), out=rgba), 6)
        print(f"{res}^3 [{name}]: nsb_rgba_on_grid {t_rgba:.3f} ms = {n / t_rgba / 1e6:.2f} Gpoints/s", flush=True)
    r.set_mlp_accumulator(abi.NSB_MLP_ACC_F16)
    t_dpng, (px, counts) = timed(lambda: r.density_png(density, R3, thresh, 4.0, False), 6)
    t_rpng, rpx = timed(lambda: r.rgba_png(rgba, R3, False), 6)
    t_dcopy, px_h = timed(lambda: px.cpu(), 6)
    t_rcopy, rpx_h = timed(lambda: rpx.cpu(), 4)
    px_h, rpx_h = px_h.numpy(), rpx_h.numpy()
    with tempfile.TemporaryDirectory() as d:
        t_denc = wall(lambda: slices.write_png(os.path.join(d, "density.png"), px_h, 1), 3)
        t_renc = wall(lambda: [slices.write_png(os.path.join(d, "%04d.png" % z), rpx_h[z], 4) for z in range(res)], 2)
    print(f"{res}^3: nsb_density_png {t_dpng:.3f} ms ({px.shape[1]}x{px.shape[0]} mosaic, counts {counts.cpu().tolist()}); nsb_rgba_png {t_rpng:.3f} ms; "
          f"device-to-host copy: mosaic {t_dcopy:.3f} ms ({px_h.nbytes / 2 ** 20:.1f} MiB), RGBA slices {t_rcopy:.3f} ms "
          f"({rpx_h.nbytes / 2 ** 20:.1f} MiB); host PNG encoding (write_png, one thread): mosaic {t_denc:.1f} ms, {res} RGBA slices {t_renc:.1f} ms",
          flush=True)
    if have_ref:
        coords = torch.empty((n, ref_slices.lib().ref_slices_coordinate_floats()), dtype=torch.float32, device="cuda")
        batch = 1 << 20
        net = torch.empty((16, batch), dtype=torch.int16, device="cuda")
        out4 = torch.empty((n, 4), dtype=torch.float32, device="cuda")
        stream = torch.cuda.current_stream().cuda_stream

        def infer_batches():
            for off in range(0, n, batch):
                k = min(batch, n - off)
                abi.check(r.lib, r.lib.nsb_inference(r.ctx, coords[off:off + k].data_ptr(), k, net.data_ptr(), batch, stream), "nsb_inference")
                out4[off:off + k] = net[:4, :k].view(torch.float16).t().float()

        t_pos, _ = timed(lambda: ref_slices.grid_coords_dev(R3, AABB, AABB, (0.0, 0.0, 1.0), coords), 6)
        t_inf, _ = timed(infer_batches, 4)
        t_cnd, _ = timed(lambda: ref_slices.compute_nerf_density_dev(out4, abi.NSB_ACT_LOGISTIC, abi.NSB_ACT_EXPONENTIAL), 6)
        ref = (f"position kernel {t_pos:.3f} ms, nsb_inference in 1M batches + cast to float4 {t_inf:.3f} ms, compute_nerf_density {t_cnd:.3f} ms; "
               f"total {t_pos + t_inf + t_cnd:.3f} ms")
        del coords, net, out4
    else:
        ref = "not measured (oracle/_ref slices build absent)"
    print(f"{res}^3: the reference's get_rgba_on_grid structure (oracle/_ref, nvcc sm_90a, fp16 accumulators): {ref}", flush=True)
    del rgba, density, px, rpx
    torch.cuda.empty_cache()
r.close()
