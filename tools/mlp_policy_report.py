"""Writes profiles/mlp_accumulator_policy.txt (measurement output, not committed): the oracle's frames under the two MLP accumulator policies (wide vs wmma __half fragments)."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from nerfshop_b200 import synthetic as syn  # noqa: E402
from oracle import oracle as orc  # noqa: E402

model = syn.make_model(seed=1337)
occ = syn.make_occupancy(model)
o = orc.Oracle(model.desc, model.params, occ)
lines = ["MLP accumulator policy: wide (double accumulate, one fp16 rounding per output) vs wmma __half accumulator fragments (round to fp16 after every k-chunk of 16)",
         "CPU oracle, synthetic fox-scale model (seed 1337), 480x270, RGBA float framebuffer (linear, premultiplied)", ""]
cams = [("fox C0", syn.fox_camera0())] + [(f"orbit {i}", syn.orbit_cameras(120)[i]) for i in (17, 57, 97)]
for name, cam in cams:
    f = syn.make_frame(model, cam, 480, 270)
    orc.set_mlp_policy(0)
    a, _, sa, _ = o.render(f)
    orc.set_mlp_policy(1)
    b, _, sb, _ = o.render(f)
    e = np.abs(a - b).max(-1)
    lines.append(f"{name:9s} L-inf {e.max():.3e}  mean {e.mean():.2e}  pixels > 1e-3: {(e > 1e-3).sum():3d} of {e.size} ({100 * (e > 1e-3).mean():.3f} %)  > 1e-4: {100 * (e > 1e-4).mean():.1f} %  "
                 f"samples {sa.n_samples} vs {sb.n_samples}")
lines += ["", "Reading: the two policies agree to ~4e-5 on average but NOT within the 1e-3 RGBA contract everywhere: 0.02 % of the pixels move by up to 1e-2",
          "(a 1-ulp change of the raw fp16 density is 0.1-0.8 % of sigma = exp(raw); it can move an early termination or the max-weight sample).",
          "The CUDA path therefore follows the reference's policy by default (fp16 wgmma accumulators) and exposes the other",
          "(nsb_set_mlp_accumulator); see DESIGN.md section 3."]
out = os.path.join(ROOT, "profiles", "mlp_accumulator_policy.txt")
os.makedirs(os.path.dirname(out), exist_ok=True)
open(out, "w").write("\n".join(lines) + "\n")
print("\n".join(lines))
