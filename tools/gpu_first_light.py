"""First-light diagnostics on a GPU box: each stage of the CUDA path against the oracle, verbosely.
Not a test (tests/ has the assertions); this prints enough to localise a failure in one gpurun trip."""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

from conftest import random_coords  # noqa: E402
from nerfshop_b200 import synthetic as syn  # noqa: E402
from nerfshop_b200.renderer import NerfRenderer  # noqa: E402
from oracle import oracle as orc  # noqa: E402

print("device", torch.cuda.get_device_name(0), torch.cuda.get_device_capability(0), flush=True)
model = syn.make_model(seed=1337)
occ = syn.make_occupancy(model)
o = orc.Oracle(model.desc, model.params, occ)
r = NerfRenderer(0)
r.upload_model(model.desc, model.params)
r.upload_occupancy(occ)
stage = sys.argv[1] if len(sys.argv) > 1 else "all"

if stage in ("all", "march"):
    f = syn.make_frame(model, syn.fox_camera0(), 160, 90)
    pix = np.arange(0, 160 * 90, 5, dtype=np.uint32)
    ro, io, co = o.march_trace(f, pix, 160)
    rg, ig, cg = r.march_trace(f, pix, 160)
    print("march: count mismatch", int((co != cg).sum()), "idx mismatch", int((io != ig).sum()), "rec bit mismatch", int((ro.view(np.uint32) != rg.view(np.uint32)).sum()),
          "of", ro.size, "total samples", int(co.sum()), flush=True)
    if (ro.view(np.uint32) != rg.view(np.uint32)).any():
        bad = np.argwhere(ro.view(np.uint32) != rg.view(np.uint32))[:5]
        for b in bad:
            print("  first diffs", b, ro[tuple(b)], rg[tuple(b)])

if stage in ("all", "encode"):
    c = random_coords(4099, seed=11)
    eo, eg = o.encode(c), r.encode(c)
    print("encode: mismatching halves", int((eo != eg).sum()), "of", eo.size, flush=True)
    if (eo != eg).any():
        bad = np.argwhere(eo != eg)[:8]
        for b in bad:
            print("  ", b, eo[tuple(b)].view(np.float16) if False else hex(int(eo[tuple(b)])), hex(int(eg[tuple(b)])))

if stage in ("all", "mlp"):
    c = random_coords(1000, seed=12)
    do = o.inference(c, density_only=True).view(np.float16).astype(np.float32)
    t0 = time.time()
    dg = r.density(c).view(np.float16).astype(np.float32)
    print("density: launched+sync in", round(time.time() - t0, 3), "s", flush=True)
    print("density: max abs err per row", np.abs(do - dg).max(1), "bit-equal frac", float((do == dg).mean()), flush=True)
    print("  oracle[:, :4]\n", do[:4, :4], "\n  gpu[:, :4]\n", dg[:4, :4])
    io_ = o.inference(c).view(np.float16).astype(np.float32)
    ig_ = r.inference(c).view(np.float16).astype(np.float32)
    print("inference: max abs err rows 0-3", np.abs(io_ - ig_)[:4].max(1), "bit-equal frac", float((io_[:4] == ig_[:4]).mean()), flush=True)
    print("  oracle[:4, :4]\n", io_[:4, :4], "\n  gpu[:4, :4]\n", ig_[:4, :4])

if stage in ("all", "render"):
    for (w, h) in ((96, 54), (320, 180)):
        f = syn.make_frame(model, syn.orbit_cameras(120)[17], w, h)
        fo, dpo, so, margin = o.render(f, want_margin=True)
        fg, dpg = r.render(f)
        st = r.stats()
        fg = fg.cpu().numpy()
        d = np.abs(fg - fo).max(-1)
        ok = margin > 2e-5
        print(f"render {w}x{h}: samples gpu {st.n_samples} oracle {so.n_samples}; hit {st.n_hit}/{so.n_hit}; alive {st.n_rays_alive}/{so.n_rays_alive}; "
              f"gpu_ms {st.gpu_ms:.3f}; Linf {d[ok].max():.3e} (all {d.max():.3e}); pixels > 1e-3: {int((d[ok] > 1e-3).sum())}; ambiguous {int((~ok).sum())}", flush=True)

if stage in ("all", "netperf"):
    n = 1 << 23
    for name, c in (("random", random_coords(n, seed=1)), ("coherent", None)):
        if c is None:  # samples along neighbouring rays: positions on a smooth 2-D sheet, sorted
            u = np.linspace(0.3, 0.6, 4096, dtype=np.float32)
            v = np.linspace(0.3, 0.5, n // 4096, dtype=np.float32)
            c = np.zeros((n, 7), np.float32)
            c[:, 0] = np.tile(u, n // 4096)
            c[:, 1] = np.repeat(v, 4096)
            c[:, 2] = 0.45 + 0.05 * np.sin(8 * c[:, 0])
            c[:, 4:] = 0.5
        ct = torch.from_numpy(c).cuda()
        n_pad = n
        out = torch.zeros((16, n_pad), dtype=torch.int16, device="cuda")
        enc = torch.zeros((32, n_pad), dtype=torch.int16, device="cuda")
        import ctypes as C
        from nerfshop_b200 import abi
        for fn, nm, dst in ((r.lib.nsb_inference, "inference", out), (r.lib.nsb_density, "density", out), (r.lib.nsb_encode, "encode", enc)):
            for rep in range(3):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                abi.check(r.lib, fn(r.ctx, ct.data_ptr(), n, dst.data_ptr(), n_pad, torch.cuda.current_stream().cuda_stream), nm)
                e1.record()
                torch.cuda.synchronize()
            ms = e0.elapsed_time(e1)
            print(f"{nm} [{name}] {n} samples: {ms:.3f} ms = {n / ms / 1e6:.2f} Gsamples/s, gather {n * 512 / ms / 1e6:.0f} GB/s algorithmic", flush=True)

if stage in ("all", "perf"):
    f = syn.make_frame(model, syn.orbit_cameras(120)[17], 1920, 1080)
    fb = torch.zeros((1080, 1920, 4), device="cuda")
    dp = torch.zeros((1080, 1920), device="cuda")
    for i in range(4):
        fb.zero_()
        r.render(f, fb, dp)
        st = r.stats()
        print(f"1080p frame {i}: {st.gpu_ms:.3f} ms, samples {st.n_samples} ({st.n_samples / st.gpu_ms / 1e6:.2f} Gsamples/s), {1920 * 1080 / st.gpu_ms / 1e3:.1f} Mrays/s, hit {st.n_hit}", flush=True)
    d = r.debug_counters()
    rounds = max(d["rounds"], 1)
    print("debug", d)
    print(f"  lane utilisation {st.n_samples / (rounds * 128):.3f}; rounds/tile {rounds / max(d['tiles'], 1):.1f}; cycles/round: acquire {d['cyc_acquire'] / rounds:.0f} encode {d['cyc_encode'] / rounds:.0f} "
          f"mlp {d['cyc_mlp'] / rounds:.0f} composite {d['cyc_composite'] / rounds:.0f}; total cyc/tile {d['cyc_total'] / max(d['tiles'], 1):.0f}", flush=True)
r.close()
