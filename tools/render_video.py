"""Renders a camera path of a NeRFshop scene to a PNG sequence: the library's version of scripts/run.py --video_camera_path.

  python tools/render_video.py --snapshot base.msgpack [--edits edits.json] --camera_path path.json --out_dir frames/
                               [--width 1920 --height 1080 --fps 60 --n_seconds 1 --spp 8 --smoothing --exposure 0]

The snapshot and the edits file are the reference's (nerfshop_b200.snapshot, nerfshop_b200.edits_io); the camera path is CameraPath::save's
JSON. Writes out_dir/%04d.png (8-bit RGBA); no video is encoded."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from nerfshop_b200 import camera_path as cp  # noqa: E402
from nerfshop_b200 import edits_io, snapshot  # noqa: E402
from nerfshop_b200 import synthetic as syn  # noqa: E402
from nerfshop_b200.renderer import NerfRenderer  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--snapshot", required=True)
    ap.add_argument("--edits", default="")
    ap.add_argument("--camera_path", required=True)
    ap.add_argument("--out_dir", required=True)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--fps", type=int, default=60)
    ap.add_argument("--n_seconds", type=int, default=1)
    ap.add_argument("--spp", type=int, default=8)
    ap.add_argument("--smoothing", action="store_true", help="camera smoothing, as run.py's --video_camera_smoothing")
    ap.add_argument("--exposure", type=float, default=0.0)
    args = ap.parse_args(argv)

    desc, params, grid, aabb_scale = snapshot.load_snapshot(args.snapshot)
    half = 0.5 * min(1 << 4, aabb_scale)  # m_aabb (testbed_nerf.cu:3410-3411)
    model = syn.SyntheticModel(desc, params, np.full(3, 0.5 - half, np.float32), np.full(3, 0.5 + half, np.float32), aabb_scale)
    r = NerfRenderer(0)
    r.upload_model(desc, params)
    r.upload_density_grid(grid)
    if args.edits:
        ops = edits_io.load_edits(args.edits, model.aabb_min, model.aabb_max)
        r.set_edit_operators([op.to_op() for op in ops])
        # membrane values: interpolate_poisson_boundary on the device, with the amplitude and switch load_edits reads (nsb_state)
        entries = [oj for oj in json.load(open(args.edits))["edit_operators"] if oj["type"] != "twist"]  # load_edits skips twist
        for i, (op, oj) in enumerate(zip(ops, entries)):
            shs = getattr(op, "cage_shs", None)
            if shs is not None:
                st = oj.get("nsb_state", {})
                r.cage_set_membrane(i, op.gamma_coordinates, shs["inside_density"], shs["outside_density"], shs["inside_shs"], shs["outside_shs"],
                                    amplitude=st.get("residual_amplitude", 1.0), apply=st.get("apply_poisson", True))
    base = syn.make_frame(model, np.eye(3, 4, dtype=np.float32), args.width, args.height, apply_operators=bool(args.edits))
    path = cp.CameraPath.load(args.camera_path)
    names = cp.render_video(r, base, path, args.n_seconds, args.fps, args.spp, args.out_dir, smoothing=args.smoothing, exposure=args.exposure)
    print(f"wrote {len(names)} frames to {args.out_dir}")
    r.close()


if __name__ == "__main__":
    main()
