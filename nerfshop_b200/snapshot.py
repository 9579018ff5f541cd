"""Reference-format snapshots (SURVEY.md §8f-3): what Testbed::save_snapshot / load_snapshot exchange
(src/testbed.cu:3054-3113): a msgpack map = the network config JSON + a "snapshot" map with
  n_params, params_type ("__half"), params_binary   <- tcnn::Trainer::serialize (external; schema as described in SURVEY
                                                       Appendix B — not verifiable in this tree)
  density_grid_size (128), density_grid_binary (float32[5*128^3]), training_step, loss, nerf.{rgb, dataset}
Two writers exist in the reference and load_snapshot here accepts both:
  save_snapshot   (testbed.cu:3090-3113): float32 grid of all 5 cascades, aabb_scale inside nerf.dataset (the whole NerfDataset, json_binding.h:140-162);
  export_snapshot (testbed.cu:3118-3183): fp16 grid of (max_cascade+1) cascades only, aabb_scale at nerf.aabb_scale, no dataset.
save_snapshot here writes the first form with the complete NerfDataset key set NerfDataset::from_json requires (json_binding.h:164-194: n_images, xforms,
render_aabb, up, offset, image_resolution, envmap_resolution, scale, aabb_scale, from_mitsuba, ...), so the reference can load the file back.
`.ingp` files are the same msgpack stream behind zstr (zlib with a gzip wrapper, `testbed.cu:168-171,3173-3176`; zstr reads plain data
through unchanged). The render path needs three things from it: the parameter block (nsb_upload_model), the density grid
(nsb_upload_density_grid -> occupancy bitfield) and aabb_scale (render/train AABB, cone angle, per_level_scale).
"""
from __future__ import annotations

import json
import os

import numpy as np

from . import abi

_BASE_CONFIG = {
    "encoding": {"otype": "HashGrid", "n_levels": 16, "n_features_per_level": 2, "log2_hashmap_size": 19, "base_resolution": 16},
    "network": {"otype": "FullyFusedMLP", "activation": "ReLU", "output_activation": "None", "n_neurons": 64, "n_hidden_layers": 1},
    "dir_encoding": {"otype": "Composite", "nested": [{"n_dims_to_encode": 3, "otype": "SphericalHarmonics", "degree": 4},
                                                       {"otype": "Identity", "n_bins": 4, "degree": 4}]},
    "rgb_network": {"otype": "FullyFusedMLP", "activation": "ReLU", "output_activation": "None", "n_neurons": 64, "n_hidden_layers": 2},
}


def save_snapshot(path: str, desc: abi.NsbModelDesc, params_u16: np.ndarray, density_grid: np.ndarray, aabb_scale: int, training_step: int = 0,
                  loss: float = 0.0, compress: bool = True) -> None:
    import msgpack

    cfg = json.loads(json.dumps(_BASE_CONFIG))
    cfg["encoding"].update({"n_levels": desc.n_levels, "n_features_per_level": desc.n_features_per_level, "log2_hashmap_size": desc.log2_hashmap_size,
                            "base_resolution": desc.base_resolution, "per_level_scale": float(desc.per_level_scale), "n_pos_dims": 3})
    p = np.ascontiguousarray(params_u16, np.uint16)
    g = np.ascontiguousarray(density_grid, np.float32).reshape(-1)
    assert g.size == abi.NSB_GRID_CELLS
    cfg["snapshot"] = {
        "n_params": int(p.size), "params_type": "__half", "params_binary": p.tobytes(),
        "density_grid_size": abi.NSB_NERF_GRIDSIZE, "density_grid_binary": g.tobytes(),
        "training_step": int(training_step), "loss": float(loss),
        "nerf": {"rgb": {"rays_per_batch": 1 << 12, "measured_batch_size": 0, "measured_batch_size_before_compaction": 0},
                 "aabb_scale": int(aabb_scale),  # where export_snapshot puts it (:3138)
                 "dataset": _dataset_json(int(aabb_scale))},
    }
    blob = msgpack.packb(cfg, use_bin_type=True)
    if path.lower().endswith(".ingp"):  # zstr::ostream: deflate with a gzip header (windowBits 15 + 16)
        import zlib

        co = zlib.compressobj(zlib.Z_DEFAULT_COMPRESSION if compress else zlib.Z_NO_COMPRESSION, zlib.DEFLATED, 15 + 16)
        blob = co.compress(blob) + co.flush()
    with open(path, "wb") as fh:
        fh.write(blob)


def _dataset_json(aabb_scale: int, scale: float = 0.33, offset=(0.5, 0.5, 0.5)) -> dict:
    """NerfDataset as to_json writes it (json_binding.h:140-162) for a snapshot without training images: every key from_json reads with .at()."""
    half = 0.5 * aabb_scale
    return {
        "n_images": 0, "paths": [], "xforms": [], "metadata": [],
        "render_aabb": {"min": [0.5 - half] * 3, "max": [0.5 + half] * 3},  # testbed_nerf.cu:3410-3411
        "up": [0.0, 1.0, 0.0], "offset": [float(v) for v in offset], "image_resolution": [0, 0], "envmap_resolution": [0, 0],
        "scale": float(scale), "aabb_scale": int(aabb_scale), "from_mitsuba": False, "is_hdr": False, "wants_importance_sampling": True,
    }


def _density_grid(blob: bytes) -> np.ndarray:
    """float32[5*128^3] from either writer: save_snapshot's float32 grid of all cascades, or export_snapshot's fp16 grid of the first max_cascade+1
    cascades (the cascades that were not exported stay 0 = empty; the bitfield step max-pools into them anyway)."""
    vol = abi.NSB_NERF_GRIDSIZE ** 3
    if len(blob) == abi.NSB_GRID_CELLS * 4:
        return np.frombuffer(blob, np.float32).copy()
    if len(blob) % (vol * 2) == 0 and 1 <= len(blob) // (vol * 2) <= abi.NSB_NERF_CASCADES:
        g = np.zeros(abi.NSB_GRID_CELLS, np.float32)
        h = np.frombuffer(blob, np.float16)
        g[: h.size] = h.astype(np.float32)
        return g
    raise abi.NsbError(f"density_grid_binary has {len(blob)} bytes: neither float32 x 5 x 128^3 (save_snapshot) nor fp16 x k x 128^3, k = 1..5 (export_snapshot)")


def _read(path: str) -> dict:
    import msgpack

    with open(path, "rb") as fh:
        blob = fh.read()
    if blob[:2] == b"\x1f\x8b" or (len(blob) > 1 and blob[0] == 0x78 and (blob[0] * 256 + blob[1]) % 31 == 0):  # zstr::istream: gzip or zlib, else plain
        import zlib

        blob = zlib.decompress(blob, 15 + 32)
    return msgpack.unpackb(blob, raw=False)


def load_dataset_transform(path: str):
    """-> (scale, offset (3 floats), from_mitsuba): the snapshot's nerf.dataset members that NerfDataset::nerf_matrix_to_ngp reads
    (nerf_loader.h:74-92), as load_snapshot restores them (json_binding.h:189-194). A snapshot without a dataset (export_snapshot's)
    leaves the NerfDataset defaults (nerf_loader.h:49-55): 1, (0, 0, 0), false."""
    ds = _read(path)["snapshot"].get("nerf", {}).get("dataset")
    if ds is None:
        return 1.0, (0.0, 0.0, 0.0), False
    return float(ds["scale"]), tuple(float(v) for v in ds["offset"]), bool(ds["from_mitsuba"])


def load_snapshot(path: str):
    """-> (NsbModelDesc, params uint16[n], density_grid float32[5*128^3], aabb_scale)."""
    cfg = _read(path)
    enc, net, rgb = cfg["encoding"], cfg["network"], cfg["rgb_network"]
    snap = cfg["snapshot"]
    if snap.get("params_type", "__half") != "__half":
        raise abi.NsbError(f"unsupported params_type {snap.get('params_type')!r} (the render path is fp16)")
    if snap.get("density_grid_size", 128) != abi.NSB_NERF_GRIDSIZE:
        raise abi.NsbError("density_grid_size must be 128")
    nerf = snap.get("nerf", {})
    if "aabb_scale" in nerf:                                    # export_snapshot (:3138)
        aabb_scale = int(nerf["aabb_scale"])
    elif "aabb_scale" in nerf.get("dataset", {}):              # save_snapshot: the whole NerfDataset
        aabb_scale = int(nerf["dataset"]["aabb_scale"])
    else:
        raise abi.NsbError("snapshot carries no aabb_scale (neither snapshot.nerf.aabb_scale nor snapshot.nerf.dataset.aabb_scale): per_level_scale and the AABB are undefined")
    pls = enc.get("per_level_scale", 0.0)
    if not pls:  # Testbed::reset_network derives it (testbed.cu:2280-2292)
        from .synthetic import per_level_scale

        pls = per_level_scale(aabb_scale, enc.get("n_levels", 16), enc.get("base_resolution", 16))
    desc = abi.NsbModelDesc(enc.get("n_levels", 16), enc.get("n_features_per_level", 2), enc.get("log2_hashmap_size", 19), enc.get("base_resolution", 16),
                            float(pls), net.get("n_neurons", 64), net.get("n_hidden_layers", 1), rgb.get("n_hidden_layers", 2), 4)
    params = np.frombuffer(snap["params_binary"], np.uint16).copy()
    if params.size != snap["n_params"]:
        raise abi.NsbError("params_binary does not hold n_params halves")
    grid = _density_grid(snap["density_grid_binary"])
    return desc, params, grid, aabb_scale
