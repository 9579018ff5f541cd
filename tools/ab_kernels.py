"""A/B timing of library builds on the 1080p orbit (4 cameras, L2 flushed, CUDA events inside nsb_render).

  python tools/ab_kernels.py name=LIBPATH ...        e.g.  base=  prof=nerfshop_b200/lib/libnerfshop_b200_prof.so   (empty LIBPATH: the product library)
Each variant runs in its own process (the library is loaded once per process). Prints fused-kernel ms (mean over the cameras), samples, debug counters
and a checksum of frame 0 (variants that must be bit-identical can be compared)."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

if len(sys.argv) > 1 and sys.argv[1] == "--child":
    sys.path.insert(0, ROOT)
    import hashlib

    import numpy as np
    import torch

    from nerfshop_b200 import synthetic as syn
    from nerfshop_b200.renderer import NerfRenderer

    W, H = int(os.environ.get("AB_W", 1920)), int(os.environ.get("AB_H", 1080))
    world = int(os.environ.get("AB_WORLD", 1))
    model = syn.make_model(seed=1337)
    occ = syn.make_occupancy(model)
    r = NerfRenderer(0)
    r.upload_model(model.desc, model.params)
    r.upload_occupancy(occ)
    cams = syn.orbit_cameras(120)
    fb = torch.zeros((H, W, 4), device="cuda")
    dp = torch.zeros((H, W), device="cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    ms, kms, smp, dbg, digest = [], [], [], None, None
    idx = [0, 30, 60, 90]
    for it in range(2 + 2 * len(idx)):
        f = syn.make_frame(model, cams[idx[it % len(idx)]], W, H, rank=0, world=world)
        flush.zero_()
        fb.zero_()
        r.render(f, fb, dp)
        st = r.stats()
        if it == 0:
            digest = hashlib.sha1(fb.cpu().numpy().tobytes()).hexdigest()[:12]
        if it >= 2:
            ms.append(st.gpu_ms)
            kms.append(st.fused_ms)
            smp.append(st.n_samples)
            dbg = r.debug_counters()
    print(json.dumps({"gpu_ms": float(np.mean(ms)), "kernel_ms": float(np.mean(kms)), "samples": float(np.mean(smp)), "Gsamples_s": float(np.mean(smp)) / float(np.mean(kms)) / 1e6,
                      "frame0_sha1": digest, "dbg_last": dbg}))
    r.close()
    sys.exit(0)

for spec in sys.argv[1:]:
    name, path = spec.split("=", 1)
    env = dict(os.environ)
    if path:
        env["NSB_LIB_PATH"] = os.path.join(ROOT, path)
    res = subprocess.run([sys.executable, os.path.abspath(__file__), "--child"], env=env, capture_output=True, text=True, timeout=600)
    line = res.stdout.strip().splitlines()[-1] if res.stdout.strip() else "FAILED: " + res.stderr[-400:]
    print(f"{name:16s} {line}", flush=True)
