"""Scores a NeRFshop snapshot against held-out views and renders screenshots: the library's version of scripts/run.py's --test_transforms
and --screenshot_transforms.

  python tools/evaluate.py --snapshot base.msgpack [--edits edits.json] --test_transforms data/transforms_test.json [--nerf_compatibility]
  python tools/evaluate.py --snapshot base.msgpack --screenshot_transforms data/transforms_test.json --screenshot_dir shots/
                           [--screenshot_frames 0 5 --screenshot_spp 16 --width 800 --height 800]

--test_transforms prints run.py's line PSNR=... [min=... max=...] SSIM=... (8 spp, black background, pixel centres, ground truth as
8-bit PNG or JPEG next to the transforms file). Screenshots are 8-bit RGBA PNG files. The snapshot and the edits file are the reference's
(nerfshop_b200.snapshot, nerfshop_b200.edits_io); the snapshot's dataset scale, offset and from_mitsuba place the cameras."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from nerfshop_b200 import edits_io, snapshot  # noqa: E402
from nerfshop_b200 import evaluate as ev  # noqa: E402
from nerfshop_b200 import synthetic as syn  # noqa: E402
from nerfshop_b200.renderer import NerfRenderer  # noqa: E402


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--snapshot", required=True)
    ap.add_argument("--edits", default="")
    ap.add_argument("--test_transforms", default="", help="NeRF-style transforms.json whose views are scored (PSNR, SSIM)")
    ap.add_argument("--screenshot_transforms", default="", help="NeRF-style transforms.json whose views are rendered to PNG files")
    ap.add_argument("--screenshot_frames", nargs="*", help="which frame(s) of --screenshot_transforms to render (default: all)")
    ap.add_argument("--screenshot_dir", default="", help="directory of the screenshots")
    ap.add_argument("--screenshot_spp", type=int, default=16)
    ap.add_argument("--width", type=int, default=0, help="screenshot width (default: the transforms file's w)")
    ap.add_argument("--height", type=int, default=0, help="screenshot height (default: the transforms file's h)")
    ap.add_argument("--nerf_compatibility", action="store_true", help="colour space sRGB and cone angle 0, as run.py's flag")
    args = ap.parse_args(argv)
    if not args.test_transforms and not args.screenshot_transforms:
        ap.error("nothing to do: give --test_transforms and/or --screenshot_transforms")

    desc, params, grid, aabb_scale = snapshot.load_snapshot(args.snapshot)
    dataset = snapshot.load_dataset_transform(args.snapshot)
    half = 0.5 * min(1 << 4, aabb_scale)  # m_aabb (testbed_nerf.cu:3410-3411)
    model = syn.SyntheticModel(desc, params, np.full(3, 0.5 - half, np.float32), np.full(3, 0.5 + half, np.float32), aabb_scale)
    r = NerfRenderer(0)
    r.upload_model(desc, params)
    r.upload_density_grid(grid)
    if args.edits:
        ops = edits_io.load_edits(args.edits, model.aabb_min, model.aabb_max)
        r.set_edit_operators([op.to_op() for op in ops])
        entries = [oj for oj in json.load(open(args.edits))["edit_operators"] if oj["type"] != "twist"]  # load_edits skips twist
        for i, (op, oj) in enumerate(zip(ops, entries)):
            shs = getattr(op, "cage_shs", None)
            if shs is not None:
                st = oj.get("nsb_state", {})
                r.cage_set_membrane(i, op.gamma_coordinates, shs["inside_density"], shs["outside_density"], shs["inside_shs"], shs["outside_shs"],
                                    amplitude=st.get("residual_amplitude", 1.0), apply=st.get("apply_poisson", True))
    base = syn.make_frame(model, np.eye(3, 4, dtype=np.float32), 64, 64, apply_operators=bool(args.edits))
    if args.nerf_compatibility:
        base.cone_angle_constant = 0.0
    if args.test_transforms:
        print("Evaluating test transforms from ", args.test_transforms)
        res = ev.evaluate(r, base, args.test_transforms, spp=8, srgb=args.nerf_compatibility, dataset=dataset)
        print(res.summary())
        base = ev.test_frame(base, args.nerf_compatibility)  # run.py's testbed keeps these settings for the screenshots
    if args.screenshot_transforms:
        names = ev.screenshots(r, base, args.screenshot_transforms, args.screenshot_dir, frames=args.screenshot_frames, spp=args.screenshot_spp,
                               width=args.width, height=args.height, dataset=dataset)
        print(f"wrote {len(names)} screenshots to {args.screenshot_dir or '.'}")
    r.close()


if __name__ == "__main__":
    main()
