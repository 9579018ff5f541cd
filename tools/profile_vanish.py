"""Cost of the cage tool's "Vanish!" (TetMesh::vanish, tet_mesh.cu:251-363): nsb_cage_vanish's device time (CUDA events around repeated
stream-ordered calls) against the wall time of the reference's own vanish on the host (oracle/_ref/libnerfshop_ref_vanish.so: 32 marking
threads, the cell list, its upload and clear_grid), for lattice cages of about 10^3, 10^4 and 10^5 tets and one whose tets reach the
coarse cascades. Every device result is checked against the reference's before it is timed.
  python tools/profile_vanish.py [--out profiles/profile_vanish.json]"""
import argparse
import json
import os
import platform
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch  # noqa: E402

import vanish_rule as vr  # noqa: E402
from nerfshop_b200 import abi, editing  # noqa: E402
from nerfshop_b200 import synthetic as syn  # noqa: E402
from nerfshop_b200.renderer import NerfRenderer  # noqa: E402

# name -> (centre, half extent, lattice n): 6 n^3 tets
CAGES = {
    "1e3": ((0.5, 0.5, 0.5), (0.2, 0.2, 0.2), 6),
    "1e4": ((0.5, 0.5, 0.5), (0.2, 0.2, 0.2), 12),
    "1e5": ((0.5, 0.5, 0.5), (0.2, 0.2, 0.2), 26),
    "coarse_1e3": ((2.6, -2.0, 2.4), (1.3, 0.9, 1.2), 6),  # outside cascades 0-1: tets dozens of cascade-2 and -3 cells wide
}


def host_info():
    cpu = platform.processor()
    try:
        with open("/proc/cpuinfo") as fh:
            cpu = next(l.split(":", 1)[1].strip() for l in fh if l.startswith("model name"))
    except (OSError, StopIteration):
        pass
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return {"cpu": cpu, "cpu_threads": os.cpu_count(), "gpu": gpu}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    model = syn.make_model(seed=1337)
    grid, _ = vr.inputs()
    info = host_info()
    print(info, flush=True)
    r = NerfRenderer(0)
    r.upload_model(model.desc, model.params)
    rows = []
    for name, (c, h, n) in CAGES.items():
        c, h = np.float32(c), np.float32(h)
        v, tets = editing.lattice_tets(c - h, c + h, n)
        op = editing.CageDeformation(model.aabb_min, model.aabb_max, *editing.box_cage(c - 1.05 * h, c + 1.05 * h), v, tets, local_rotations=False)
        op.vertices = v
        op.lut_offsets = np.zeros(abi.NSB_GRID_CELLS + 1, np.uint32)
        op.lut_idx = op._grid(op.vertices, op.lut_offsets, None)
        r.set_edit_operators([op.to_op()])
        bits = r.upload_density_grid(grid)
        n_cleared = r.cage_vanish(0, count=True)
        g_dev, b_dev = r.download_density_grid()
        # the reference's vanish on the same grid and bitfield: best of two runs
        ref_s, stored = [], None
        for _ in range(2):
            stored = vr.reference_vanish(v, v, tets, model.aabb_min, model.aabb_max, grid, bits)
            ref_s.append(vr.reference_vanish.seconds)
        g_ref, b_ref = vr.apply_stored(grid, stored)
        assert np.array_equal(g_dev.view(np.uint32), g_ref.view(np.uint32)) and np.array_equal(b_dev, b_ref), name
        # the device call: uncounted (stream-ordered) calls back to back, after a warm-up
        st = torch.cuda.current_stream().cuda_stream
        for _ in range(3):
            r.cage_vanish(0, stream=st)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            r.cage_vanish(0, stream=st)
        e1.record()
        torch.cuda.synchronize()
        dev_ms = e0.elapsed_time(e1) / args.reps
        touched = vr.touched_cells(v, tets).reshape(5, -1).sum(1)
        row = {"cage": name, "tets": int(tets.shape[0]), "cells_touched_per_cascade": touched.tolist(), "cells_changed": n_cleared,
               "device_ms": dev_ms, "reference_host_ms": min(ref_s) * 1e3, "speedup": min(ref_s) * 1e3 / dev_ms}
        print(json.dumps(row), flush=True)
        rows.append(row)
    r.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump({"host": info, "rows": rows}, fh, indent=1)


if __name__ == "__main__":
    main()
