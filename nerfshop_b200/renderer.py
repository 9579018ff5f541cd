"""Python host mirror of the reference surfaces the render path is called through, over the C ABI.

  NerfRenderer.render            <- Testbed::render_nerf            (testbed_nerf.cu:3066)
  NerfRenderer.render_to_cpu     <- Testbed::render_to_cpu          (python_api.cu:129-175)
  NerfRenderer.inference / density <- NerfNetwork::inference_mixed_precision / ::density
  NerfRenderer.map_rays / poisson_residuals <- EditOperator::map_rays / ::compute_poisson_full_residuals
  NerfRenderer.{add,reset}_edit_operator <- NerfTracer::{add,reset}_edit_operator (testbed.h:129-240)
  NerfRenderer.density_on_grid / marching_cubes / mesh_shade / mesh_download <- Testbed::marching_cubes (testbed_nerf.cu:4614-4649);
      nerfshop_b200.mesh builds the reference's Python-facing calls on them
  NerfRenderer.rgba_on_grid / density_png / rgba_png <- Testbed::get_rgba_on_grid (testbed_nerf.cu:4588-4612) and the pixel loops of
      save_density_grid_to_png / save_rgba_grid_to_png_sequence (marching_cubes.cu:898-1015); nerfshop_b200.slices writes the files
  NerfRenderer.render_accumulate / frame_to_rgba8 <- Testbed::render_to_cpu's sub-frame loop (python_api.cu:129-175) and scripts/run.py's
      8-bit video frames (write_image, scripts/common.py:122-178); nerfshop_b200.camera_path builds camera paths and videos on them
  NerfRenderer.reference_image / image_metrics <- scripts/run.py's --test_transforms block (run.py:215-302): read_image's ground truth and
      compute_error("MSE" / "SSIM") with their means; nerfshop_b200.evaluate scores test views and writes screenshots on them

torch is used for device memory and streams only; every computation is a call into libnerfshop_b200.so.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import abi, slices


def _torch():
    import torch

    return torch


def _grid_query(res3d, aabb, train_aabb) -> abi.NsbGridQuery:
    """The NsbGridQuery of density_on_grid and rgba_on_grid: res3d points over aabb, warped with train_aabb."""
    q = abi.NsbGridQuery()
    q.res[:] = [int(v) for v in res3d]
    q.aabb_min[:], q.aabb_max[:] = [float(v) for v in aabb[0]], [float(v) for v in aabb[1]]
    q.train_aabb_min[:], q.train_aabb_max[:] = [float(v) for v in train_aabb[0]], [float(v) for v in train_aabb[1]]
    return q


class NerfRenderer:
    def __init__(self, device: int | None = None):
        torch = _torch()
        if not torch.cuda.is_available():
            raise abi.NsbError("no CUDA device: nerfshop_b200 has no CPU fallback")
        self.lib = abi.load_library()
        self.device = torch.cuda.current_device() if device is None else device
        self.ctx = C.c_void_p()
        abi.check(self.lib, self.lib.nsb_create(self.device, C.byref(self.ctx)), "nsb_create")
        self._ops = []
        self._keep = None

    def close(self):
        if self.ctx:
            self.lib.nsb_destroy(self.ctx)
            self.ctx = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- state -------------------------------------------------------------------------------------
    def upload_model(self, desc: abi.NsbModelDesc, params_u16: np.ndarray):
        p = np.ascontiguousarray(params_u16, dtype=np.uint16)
        abi.check(self.lib, self.lib.nsb_upload_model(self.ctx, C.byref(desc), p.ctypes.data, p.size), "nsb_upload_model")

    def set_mlp_accumulator(self, policy: int):
        """NSB_MLP_ACC_F16 (default: the arithmetic of tiny-cuda-nn's wmma __half accumulator fragments) or NSB_MLP_ACC_F32."""
        abi.check(self.lib, self.lib.nsb_set_mlp_accumulator(self.ctx, int(policy)), "nsb_set_mlp_accumulator")

    def upload_occupancy(self, bitfield: np.ndarray):
        b = np.ascontiguousarray(bitfield, dtype=np.uint8)
        abi.check(self.lib, self.lib.nsb_upload_occupancy(self.ctx, b.ctypes.data, b.size), "nsb_upload_occupancy")

    def upload_density_grid(self, density_grid: np.ndarray) -> np.ndarray:
        """Snapshot path: float[5*128^3] density grid -> occupancy bitfield (returned) — update_density_grid_mean_and_bitfield."""
        g = np.ascontiguousarray(density_grid, dtype=np.float32).reshape(-1)
        out = np.zeros(abi.NSB_BITFIELD_BYTES, np.uint8)
        abi.check(self.lib, self.lib.nsb_upload_density_grid(self.ctx, g.ctypes.data, g.size, out.ctypes.data), "nsb_upload_density_grid")
        return out

    def update_density_grid(self, rng, ema_step: int, n_uniform: int, n_nonuniform: int = 0, reset_grid: bool = False, n_cascades: int = 3,
                            decay: float = 0.95, train_aabb=((-1.5, -1.5, -1.5), (2.5, 2.5, 2.5)), density_activation: int = abi.NSB_ACT_EXPONENTIAL,
                            apply_operators: bool = True, stream: int = 0) -> None:
        """Testbed::update_density_grid_nerf_operator (testbed_nerf.cu:3533-3639): one update of the context's running density
        grid and occupancy bitfield through the uploaded operators. `rng` (nerfshop_b200.rng.Pcg32) is advanced like m_rng."""
        u = abi.NsbGridUpdate()
        u.n_uniform_samples, u.n_nonuniform_samples = int(n_uniform), int(n_nonuniform)
        u.reset_grid, u.n_cascades, u.decay, u.ema_step = int(bool(reset_grid)), int(n_cascades), float(decay), int(ema_step)
        u.rng_state, u.rng_inc = rng.state, rng.inc
        u.train_aabb_min[:] = train_aabb[0]
        u.train_aabb_max[:] = train_aabb[1]
        u.density_activation, u.apply_operators = int(density_activation), int(bool(apply_operators))
        abi.check(self.lib, self.lib.nsb_update_density_grid(self.ctx, C.byref(u), stream), "nsb_update_density_grid")
        rng.advance()  # :3576
        rng.advance()  # :3589
        return u

    def update_density_grid_nerf_render(self, state: dict, n_iterations: int, reset_grid: bool, **kw) -> None:
        """Testbed::update_density_grid_nerf_render (testbed_nerf.cu:3514-3520): full-grid uniform updates after an edit.
        `state` carries Testbed's members {"rng": Pcg32, "ema_step": int, "max_cascade": int}."""
        n_casc = state["max_cascade"] + 1
        for i in range(n_iterations):
            self.update_density_grid(state["rng"], state["ema_step"], 128 ** 3 * n_casc, 0, reset_grid and i == 0, n_cascades=n_casc, **kw)
            state["ema_step"] += 1  # :3636
        _torch().cuda.synchronize(self.device)

    def download_density_grid(self, want_grid: bool = True, want_bitfield: bool = True):
        grid = np.zeros(abi.NSB_GRID_CELLS, np.float32) if want_grid else None
        bits = np.zeros(abi.NSB_BITFIELD_BYTES, np.uint8) if want_bitfield else None
        abi.check(self.lib, self.lib.nsb_download_density_grid(self.ctx, None if grid is None else grid.ctypes.data, None if bits is None else bits.ctypes.data),
                  "nsb_download_density_grid")
        return grid, bits

    # ---- per-edit rebuild on the device (GrowingSelection::update_tet_mesh, growing_selection.cu:1615) ----
    def cage_attach_mvc(self, op_index: int, mvc_weights: np.ndarray) -> None:
        w = np.ascontiguousarray(mvc_weights, np.float32)
        abi.check(self.lib, self.lib.nsb_cage_attach_mvc(self.ctx, op_index, w.ctypes.data, w.shape[1]), "nsb_cage_attach_mvc")

    def cage_deform(self, op_index: int, cage_vertices: np.ndarray, stream: int = 0) -> None:
        cv = np.ascontiguousarray(cage_vertices, np.float32).reshape(-1, 3)
        abi.check(self.lib, self.lib.nsb_cage_deform(self.ctx, op_index, cv.ctypes.data, cv.shape[0], stream), "nsb_cage_deform")

    def cage_vanish(self, op_index: int, count: bool = False, stream: int = 0):
        """TetMesh::vanish (tet_mesh.cu:251-363): zero the density and clear the occupancy bit of every cell, at every cascade, that the
        cage operator's current tets touch. Stream-ordered; with count=True it synchronises and returns the number of cells whose density or
        bit changed. A later update_density_grid refills the cells from the network."""
        n = C.c_uint64()
        abi.check(self.lib, self.lib.nsb_cage_vanish(self.ctx, op_index, C.byref(n) if count else None, stream), "nsb_cage_vanish")
        return int(n.value) if count else None

    def cage_download(self, op_index: int, n_vertices: int, n_tets: int, rotations: bool = True) -> dict:
        n = C.c_uint64()
        abi.check(self.lib, self.lib.nsb_cage_download(self.ctx, op_index, None, None, None, None, 0, C.byref(n), None), "nsb_cage_download")
        out = dict(vertices=np.zeros((n_vertices, 3), np.float32), rotations=np.zeros((n_tets, 9), np.float32) if rotations else None,
                   lut_offsets=np.zeros(abi.NSB_GRID_CELLS + 1, np.uint32), lut_idx=np.zeros(max(int(n.value), 1), np.uint32), boxes=np.zeros(12, np.float32))
        abi.check(self.lib, self.lib.nsb_cage_download(self.ctx, op_index, out["vertices"].ctypes.data, out["rotations"].ctypes.data if rotations else None,
                                                       out["lut_offsets"].ctypes.data, out["lut_idx"].ctypes.data, out["lut_idx"].size, C.byref(n),
                                                       out["boxes"].ctypes.data), "nsb_cage_download")
        out["lut_idx"] = out["lut_idx"][: int(n.value)]
        return out

    # ---- membrane boundary values (GrowingSelection::compute_poisson_boundary / interpolate_poisson_boundary) ----
    def poisson_boundary(self, points: np.ndarray, is_inside: bool, seed: int = 0, sampling_width: int = 10, hemisphere_width: int = 10,
                         train_aabb=((-1.5, -1.5, -1.5), (2.5, 2.5, 2.5)), rgb_activation: int = abi.NSB_ACT_LOGISTIC,
                         density_activation: int = abi.NSB_ACT_EXPONENTIAL):
        pts = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
        p = abi.NsbBoundarySampling()
        p.sampling_width, p.hemisphere_width, p.seed = sampling_width, hemisphere_width, seed
        p.train_aabb_min[:] = train_aabb[0]
        p.train_aabb_max[:] = train_aabb[1]
        p.rgb_activation, p.density_activation, p.is_inside = rgb_activation, density_activation, int(is_inside)
        dens, shs = np.zeros(pts.shape[0], np.float32), np.zeros((pts.shape[0], 27), np.float32)
        abi.check(self.lib, self.lib.nsb_poisson_boundary(self.ctx, pts.ctypes.data, pts.shape[0], C.byref(p), dens.ctypes.data, shs.ctypes.data), "nsb_poisson_boundary")
        return dens, shs, p

    def cage_set_membrane(self, op_index: int, gamma: np.ndarray, inside_density, outside_density, inside_shs, outside_shs, amplitude: float = 1.0,
                          apply: bool = True):
        g = np.ascontiguousarray(gamma, np.float32)
        arrs = [np.ascontiguousarray(a, np.float32) for a in (inside_density, outside_density, inside_shs, outside_shs)]
        nv = g.shape[0]
        b_shs, b_od, b_rd = np.zeros((nv, 27), np.float32), np.zeros(nv, np.float32), np.zeros(nv, np.float32)
        abi.check(self.lib, self.lib.nsb_cage_set_membrane(self.ctx, op_index, g.ctypes.data, g.shape[1], *[a.ctypes.data for a in arrs], float(amplitude), int(apply),
                                                           b_shs.ctypes.data, b_od.ctypes.data, b_rd.ctypes.data), "nsb_cage_set_membrane")
        return b_shs, b_od, b_rd

    def set_edit_operators(self, ops):
        """ops: list of (NsbEditOp, keepalive) in m_edit_operators order."""
        self._ops = list(ops or [])
        if self._ops:
            arr = (abi.NsbEditOp * len(self._ops))(*[o[0] for o in self._ops])
            abi.check(self.lib, self.lib.nsb_set_edit_ops(self.ctx, arr, len(self._ops)), "nsb_set_edit_ops")
        else:
            abi.check(self.lib, self.lib.nsb_set_edit_ops(self.ctx, None, 0), "nsb_set_edit_ops")

    def add_edit_operator(self, op):
        self.set_edit_operators(self._ops + [op])

    def reset_edit_operators(self):
        self.set_edit_operators([])

    # ---- the hot path ------------------------------------------------------------------------------------
    def render(self, frame: abi.NsbFrame, fb=None, depth=None, stream=None):
        """fb: float32 CUDA tensor [H, W, 4] (over-blended onto, like render_buffer.frame_buffer()); depth [H, W]."""
        torch = _torch()
        dev = torch.device("cuda", self.device)
        if fb is None:
            fb = torch.zeros((frame.height, frame.width, 4), dtype=torch.float32, device=dev)
        if depth is None:
            depth = torch.zeros((frame.height, frame.width), dtype=torch.float32, device=dev)
        s = torch.cuda.current_stream(dev).cuda_stream if stream is None else stream
        abi.check(self.lib, self.lib.nsb_render(self.ctx, C.byref(frame), fb.data_ptr(), depth.data_ptr(), s), "nsb_render")
        return fb, depth

    def render_to_cpu(self, frame: abi.NsbFrame, fb_host=None, depth_host=None):
        """Host-buffer entry point (pinned torch tensors or numpy arrays)."""
        if fb_host is None:
            fb_host = np.zeros((frame.height, frame.width, 4), np.float32)
        if depth_host is None:
            depth_host = np.zeros((frame.height, frame.width), np.float32)
        fp = fb_host.data_ptr() if hasattr(fb_host, "data_ptr") else fb_host.ctypes.data
        dp = depth_host.data_ptr() if hasattr(depth_host, "data_ptr") else depth_host.ctypes.data
        abi.check(self.lib, self.lib.nsb_render_host(self.ctx, C.byref(frame), fp, dp), "nsb_render_host")
        return fb_host, depth_host

    def render_to_cpu_async(self, frame: abi.NsbFrame, fb_host, depth_host=None) -> int:
        """nsb_render_host_async: returns a ticket; fb_host / depth_host (pinned) are valid after wait_host_frame(ticket). The copy of this frame
        overlaps the render of the next one."""
        fp = fb_host.data_ptr() if hasattr(fb_host, "data_ptr") else fb_host.ctypes.data
        dp = None if depth_host is None else (depth_host.data_ptr() if hasattr(depth_host, "data_ptr") else depth_host.ctypes.data)
        ticket = C.c_uint64()
        abi.check(self.lib, self.lib.nsb_render_host_async(self.ctx, C.byref(frame), fp, dp, C.byref(ticket)), "nsb_render_host_async")
        return ticket.value

    def wait_host_frame(self, ticket: int) -> None:
        abi.check(self.lib, self.lib.nsb_host_frame_wait(self.ctx, ticket), "nsb_host_frame_wait")

    def stats(self) -> abi.NsbRenderStats:
        st = abi.NsbRenderStats()
        abi.check(self.lib, self.lib.nsb_get_stats(self.ctx, C.byref(st)), "nsb_get_stats")
        return st

    def debug_counters(self) -> dict:
        out = (C.c_uint64 * 7)()
        abi.check(self.lib, self.lib.nsb_debug_counters(self.ctx, out, 7), "nsb_debug_counters")
        keys = ("rounds", "cyc_acquire", "cyc_encode", "cyc_mlp", "cyc_composite", "cyc_total", "tiles")  # summed over / counting render tiles
        return dict(zip(keys, [int(v) for v in out]))

    # ---- multi-GPU framebuffer shards ------------------------------------------------------------------
    def tiles_for_rank(self, width, height, rank, world) -> int:
        n = C.c_uint32()
        abi.check(self.lib, self.lib.nsb_tiles_for_rank(width, height, rank, world, C.byref(n)), "nsb_tiles_for_rank")
        return n.value

    def pack_tiles(self, fb, depth, rank, world, out_rgba, out_depth=None):
        torch = _torch()
        H, W = fb.shape[0], fb.shape[1]
        s = torch.cuda.current_stream().cuda_stream
        abi.check(self.lib, self.lib.nsb_pack_tiles(self.ctx, fb.data_ptr(), 0 if depth is None else depth.data_ptr(), W, H, rank, world,
                                                    out_rgba.data_ptr(), 0 if out_depth is None else out_depth.data_ptr(), s), "nsb_pack_tiles")

    def unpack_tiles(self, packed_rgba, packed_depth, rank, world, fb, depth=None):
        torch = _torch()
        H, W = fb.shape[0], fb.shape[1]
        s = torch.cuda.current_stream().cuda_stream
        abi.check(self.lib, self.lib.nsb_unpack_tiles(self.ctx, packed_rgba.data_ptr(), 0 if packed_depth is None else packed_depth.data_ptr(), W, H, rank, world,
                                                      fb.data_ptr(), 0 if depth is None else depth.data_ptr(), s), "nsb_unpack_tiles")

    def unpack_gathered(self, gathered_rgba, gathered_depth, rank_stride_floats, skip_rank, world, fb, depth=None):
        """ONE launch: every rank's packed tiles of an all-gather result (rank k's float4 tiles at gathered_rgba + k*stride, its depth floats at
        gathered_depth + k*stride) except skip_rank's -> fb (+ depth)."""
        torch = _torch()
        H, W = fb.shape[0], fb.shape[1]
        s = torch.cuda.current_stream().cuda_stream
        abi.check(self.lib, self.lib.nsb_unpack_gathered(self.ctx, gathered_rgba.data_ptr(), 0 if gathered_depth is None else gathered_depth.data_ptr(), W, H, skip_rank, world,
                                                         int(rank_stride_floats), fb.data_ptr(), 0 if depth is None else depth.data_ptr(), s), "nsb_unpack_gathered")

    # ---- frame post-process (CudaRenderBuffer::accumulate / ::tonemap) ---------------------------------------
    def accumulate(self, frame_buffer, accumulate_buffer, spp: int, color_space: int = abi.NSB_COLOR_LINEAR):
        torch = _torch()
        H, W = frame_buffer.shape[0], frame_buffer.shape[1]
        abi.check(self.lib, self.lib.nsb_accumulate(self.ctx, frame_buffer.data_ptr(), accumulate_buffer.data_ptr(), W, H, spp, color_space,
                                                    torch.cuda.current_stream().cuda_stream), "nsb_accumulate")

    def tonemap(self, accumulate_buffer, params: "abi.NsbTonemap", out=None):
        torch = _torch()
        H, W = accumulate_buffer.shape[0], accumulate_buffer.shape[1]
        if out is None:
            out = torch.empty_like(accumulate_buffer)
        abi.check(self.lib, self.lib.nsb_tonemap(self.ctx, accumulate_buffer.data_ptr(), out.data_ptr(), W, H, C.byref(params),
                                                 torch.cuda.current_stream().cuda_stream), "nsb_tonemap")
        return out

    # ---- whole output frames (Testbed::render_to_cpu's sub-frame loop, scripts/run.py's 8-bit frames) ------------------------------
    def render_accumulate(self, frames, tonemap: "abi.NsbTonemap", accumulate=None, out=None, stream=None):
        """nsb_render_accumulate: every sub-frame rendered and accumulated (spp = its spp_index), then one tonemap. frames: NsbFrames of one
        size; accumulate / out: float32 CUDA tensors [H, W, 4] (allocated if None). Returns (accumulate, out). Stream-ordered."""
        torch = _torch()
        frames = list(frames)
        if not frames:
            raise ValueError("render_accumulate: no sub-frames")
        H, W = frames[0].height, frames[0].width
        dev = torch.device("cuda", self.device)
        if accumulate is None:
            accumulate = torch.empty((H, W, 4), dtype=torch.float32, device=dev)
        if out is None:
            out = torch.empty((H, W, 4), dtype=torch.float32, device=dev)
        arr = (abi.NsbFrame * len(frames))(*frames)
        s = torch.cuda.current_stream(dev).cuda_stream if stream is None else stream
        abi.check(self.lib, self.lib.nsb_render_accumulate(self.ctx, arr, len(frames), C.byref(tonemap), accumulate.data_ptr(), out.data_ptr(), s),
                  "nsb_render_accumulate")
        return accumulate, out

    def frame_to_rgba8(self, rgba, exposure: float = 0.0, n_channels: int = 4, out=None, stream=None):
        """nsb_frame_to_rgba8 on a float32 CUDA tensor [H, W, 4] of linear premultiplied RGBA: run.py's np.clip(frame * 2**exposure, 0, 1)
        and write_image's 8-bit pixels, uint8 CUDA tensor [H, W, n_channels] (3: RGB without alpha). Stream-ordered."""
        torch = _torch()
        H, W = rgba.shape[0], rgba.shape[1]
        if out is None:
            out = torch.empty((H, W, n_channels), dtype=torch.uint8, device=torch.device("cuda", self.device))
        s = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        abi.check(self.lib, self.lib.nsb_frame_to_rgba8(self.ctx, rgba.data_ptr(), W, H, float(exposure), int(n_channels), out.data_ptr(), s),
                  "nsb_frame_to_rgba8")
        return out

    # ---- image-quality metrics (scripts/run.py --test_transforms) ------------------------------------------------------------------
    def reference_image(self, pixels, srgb_blend: bool = False, background=(0.0, 0.0, 0.0, 1.0), out=None, stream=None):
        """nsb_reference_image: read_image's linear premultiplied RGBA (alpha 1 for RGB) from decoded 8-bit pixels, uint8 CUDA tensor
        [H, W, 3 or 4]; srgb_blend: run.py's blend over `background` in sRGB (RGBA only). Returns float32 CUDA tensor [H, W, 4]. Stream-ordered."""
        torch = _torch()
        H, W, nc = pixels.shape
        if out is None:
            out = torch.empty((H, W, 4), dtype=torch.float32, device=torch.device("cuda", self.device))
        bg = (C.c_float * 4)(*[float(v) for v in background])
        s = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        abi.check(self.lib, self.lib.nsb_reference_image(self.ctx, pixels.data_ptr(), W, H, nc, int(bool(srgb_blend)), bg, out.data_ptr(), s),
                  "nsb_reference_image")
        return out

    def image_metrics(self, image, ref, out=None, mse_map=None, ssim_map=None, stream=None):
        """nsb_image_metrics on two float32 CUDA tensors [H, W, 4] (the rendered frame, the ground truth): run.py's MSE and SSIM of the frame,
        float32 CUDA tensor [2] = (MSE, SSIM), left on the device. mse_map / ssim_map: float32 CUDA tensors [H, W] to receive the maps, or
        None. Stream-ordered."""
        torch = _torch()
        H, W = image.shape[0], image.shape[1]
        if tuple(ref.shape[:2]) != (H, W):
            raise ValueError(f"image_metrics: image {tuple(image.shape)} and ground truth {tuple(ref.shape)} differ in size")
        if out is None:
            out = torch.empty(2, dtype=torch.float32, device=torch.device("cuda", self.device))
        s = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        abi.check(self.lib, self.lib.nsb_image_metrics(self.ctx, image.data_ptr(), ref.data_ptr(), W, H, out.data_ptr(),
                                                       0 if mse_map is None else mse_map.data_ptr(), 0 if ssim_map is None else ssim_map.data_ptr(), s),
                  "nsb_image_metrics")
        return out

    # ---- operator-level entry points ---------------------------------------------------------------------
    def _coords(self, coords):
        torch = _torch()
        c = torch.as_tensor(np.ascontiguousarray(coords, np.float32)) if not hasattr(coords, "data_ptr") else coords
        return c.to(torch.device("cuda", self.device)).contiguous()

    def _run_net(self, fn, name, coords, rows):
        torch = _torch()
        c = self._coords(coords)
        n = c.shape[0]
        n_pad = ((n + 127) // 128) * 128
        if n == 0:
            abi.check(self.lib, fn(self.ctx, None, 0, None, 0, None), name)  # empty batch is a no-op
            return np.zeros((rows, 0), np.uint16)
        out = torch.zeros((rows, n_pad), dtype=torch.int16, device=c.device)
        abi.check(self.lib, fn(self.ctx, c.data_ptr(), n, out.data_ptr(), n_pad, torch.cuda.current_stream().cuda_stream), name)
        torch.cuda.synchronize()
        return out.cpu().numpy().view(np.uint16)[:, :n]

    def inference(self, coords) -> np.ndarray:
        return self._run_net(self.lib.nsb_inference, "nsb_inference", coords, 16)

    def density(self, coords) -> np.ndarray:
        return self._run_net(self.lib.nsb_density, "nsb_density", coords, 16)

    def encode(self, coords) -> np.ndarray:
        return self._run_net(self.lib.nsb_encode, "nsb_encode", coords, 32)

    def map_rays(self, coords):
        torch = _torch()
        c = self._coords(coords).clone()
        n = c.shape[0]
        mask = torch.zeros(n, dtype=torch.uint8, device=c.device)
        abi.check(self.lib, self.lib.nsb_map_rays(self.ctx, c.data_ptr(), mask.data_ptr(), n, torch.cuda.current_stream().cuda_stream), "nsb_map_rays")
        torch.cuda.synchronize()
        return c.cpu().numpy(), mask.cpu().numpy()

    def poisson_residuals(self, coords):
        torch = _torch()
        c = self._coords(coords)
        n = c.shape[0]
        sh = torch.zeros((n, 27), dtype=torch.float32, device=c.device)
        od = torch.zeros(n, dtype=torch.float32, device=c.device)
        rd = torch.zeros(n, dtype=torch.float32, device=c.device)
        abi.check(self.lib, self.lib.nsb_poisson_residuals(self.ctx, c.data_ptr(), n, sh.data_ptr(), od.data_ptr(), rd.data_ptr(),
                                                           torch.cuda.current_stream().cuda_stream), "nsb_poisson_residuals")
        torch.cuda.synchronize()
        return sh.cpu().numpy(), od.cpu().numpy(), rd.cpu().numpy()

    def march_trace(self, frame: abi.NsbFrame, pixels: np.ndarray, max_samples: int):
        torch = _torch()
        dev = torch.device("cuda", self.device)
        p = torch.as_tensor(np.ascontiguousarray(pixels, np.uint32).view(np.int32)).to(dev)
        n = p.numel()
        rec = torch.zeros((n, max_samples, 5), dtype=torch.float32, device=dev)
        idx = torch.zeros((n, max_samples, 2), dtype=torch.int32, device=dev)
        cnt = torch.zeros(n, dtype=torch.int32, device=dev)
        abi.check(self.lib, self.lib.nsb_march_trace(self.ctx, C.byref(frame), p.data_ptr(), n, max_samples, rec.data_ptr(), idx.data_ptr(), cnt.data_ptr(),
                                                     torch.cuda.current_stream().cuda_stream), "nsb_march_trace")
        torch.cuda.synchronize()
        return rec.cpu().numpy(), idx.cpu().numpy().view(np.uint32), cnt.cpu().numpy().view(np.uint32)

    # ---- mesh extraction (Testbed::marching_cubes, testbed_nerf.cu:4614-4649) -----------------------------------------------
    def density_on_grid(self, res3d, aabb, train_aabb, out=None, stream=None):
        """Testbed::get_density_on_grid: float32 CUDA tensor [res_z, res_y, res_x] (x fastest) of raw densities, -10000 where the running
        density grid is empty. res3d: positive multiples of 16."""
        torch = _torch()
        q = _grid_query(res3d, aabb, train_aabb)
        if out is None:
            out = torch.empty((max(q.res[2], 0), max(q.res[1], 0), max(q.res[0], 0)), dtype=torch.float32, device=torch.device("cuda", self.device))
        s = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        abi.check(self.lib, self.lib.nsb_density_on_grid(self.ctx, C.byref(q), out.data_ptr(), s), "nsb_density_on_grid")
        return out

    def marching_cubes(self, density, res3d, aabb, thresh: float, stream=None):
        """marching_cubes_gpu on a float32 CUDA tensor of res3d points (x fastest): (n_vertices, n_indices) of the mesh the context now holds."""
        torch = _torch()
        res = (C.c_int32 * 3)(*[int(v) for v in res3d])
        mn, mx = (C.c_float * 3)(*[float(v) for v in aabb[0]]), (C.c_float * 3)(*[float(v) for v in aabb[1]])
        nv, ni = C.c_uint64(), C.c_uint64()
        s = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        abi.check(self.lib, self.lib.nsb_marching_cubes(self.ctx, density.data_ptr(), res, mn, mx, float(thresh), C.byref(nv), C.byref(ni), s), "nsb_marching_cubes")
        return nv.value, ni.value

    def mesh_shade(self, train_aabb, rgb_activation: int = abi.NSB_ACT_LOGISTIC, linear_colors: bool = False, stream=None):
        """Vertex normals (compute_mesh_1ring) and colours (compute_mesh_vertex_colors) of the context's mesh."""
        torch = _torch()
        mn, mx = (C.c_float * 3)(*[float(v) for v in train_aabb[0]]), (C.c_float * 3)(*[float(v) for v in train_aabb[1]])
        s = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        abi.check(self.lib, self.lib.nsb_mesh_shade(self.ctx, mn, mx, int(rgb_activation), int(bool(linear_colors)), s), "nsb_mesh_shade")

    # ---- mesh optimisation (Testbed::optimise_mesh_step, testbed_nerf.cu:4470-4513) ---------------------------------------------
    def density_gradient(self, coords, want_dfeat: bool = False):
        """NerfNetwork::density + input_gradient(3) on NerfCoordinate rows: (grad float32 [n, 3] w.r.t. the warped position, raw density
        fp16 bits uint16 [n][, dL/dfeatures * 128 as fp16 bits uint16 [32, n]])."""
        torch = _torch()
        c = self._coords(coords)
        n = c.shape[0]
        n_pad = ((n + 127) // 128) * 128
        grad = torch.zeros((n, 3), dtype=torch.float32, device=c.device)
        dens = torch.zeros(n_pad, dtype=torch.int16, device=c.device)
        dfeat = torch.zeros((32, n_pad), dtype=torch.int16, device=c.device) if want_dfeat else None
        abi.check(self.lib, self.lib.nsb_density_gradient(self.ctx, c.data_ptr() if n else None, n, grad.data_ptr() if n else None, 3,
                                                          dens.data_ptr() if n else None, dfeat.data_ptr() if (want_dfeat and n) else None, n_pad,
                                                          torch.cuda.current_stream().cuda_stream), "nsb_density_gradient")
        torch.cuda.synchronize()
        out = (grad.cpu().numpy(), dens.cpu().numpy().view(np.uint16)[:n])
        return out + (dfeat.cpu().numpy().view(np.uint16)[:, :n],) if want_dfeat else out

    def mesh_optimise(self, n_steps: int, thresh: float, train_aabb, smooth_amount: float = 2048.0, density_amount: float = 128.0,
                      inflate_amount: float = 1.0, stream=None):
        """n_steps of Testbed::optimise_mesh_step on the context's mesh (its vertex rows move in place; read them with mesh_download)."""
        torch = _torch()
        p = abi.NsbMeshOptimise()
        p.thresh, p.smooth_amount, p.density_amount, p.inflate_amount = float(thresh), float(smooth_amount), float(density_amount), float(inflate_amount)
        p.train_aabb_min[:], p.train_aabb_max[:] = [float(v) for v in train_aabb[0]], [float(v) for v in train_aabb[1]]
        s = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        abi.check(self.lib, self.lib.nsb_mesh_optimise(self.ctx, C.byref(p), int(n_steps), s), "nsb_mesh_optimise")

    def mesh_download(self, n_vertices: int, n_indices: int, padded: bool = True, shaded: bool = True) -> dict:
        """The mesh as numpy arrays: V, N (not normalised), C with n_vertices rows (rounded up to 128 when padded, as the reference
        allocates them), F [n_indices / 3, 3] uint32."""
        rows = ((n_vertices + 127) // 128) * 128 if padded else n_vertices
        V = np.zeros((rows, 3), np.float32)
        N = np.zeros((rows, 3), np.float32) if shaded else None
        Cc = np.zeros((rows, 3), np.float32) if shaded else None
        F = np.zeros((n_indices // 3, 3), np.uint32)
        abi.check(self.lib, self.lib.nsb_mesh_download(self.ctx, V.ctypes.data, None if N is None else N.ctypes.data, None if Cc is None else Cc.ctypes.data,
                                                       rows, F.ctypes.data, F.size), "nsb_mesh_download")
        return dict(V=V, N=N, C=Cc, F=F)

    # ---- density and RGBA slices (the export panel, testbed.cu:952-966) -----------------------------------------------------------
    def rgba_on_grid(self, res3d, aabb, train_aabb, ray_dir, rgb_activation: int = abi.NSB_ACT_LOGISTIC,
                     density_activation: int = abi.NSB_ACT_EXPONENTIAL, out=None, stream=None):
        """Testbed::get_rgba_on_grid: float32 CUDA tensor [res_z, res_y, res_x, 4] (x fastest) of compute_nerf_density's premultiplied
        rgb and alpha, the network seen from ray_dir at the grid positions of density_on_grid over aabb. res3d: positive multiples of 16."""
        torch = _torch()
        q = _grid_query(res3d, aabb, train_aabb)
        d = (C.c_float * 3)(*[float(v) for v in ray_dir])
        if out is None:
            out = torch.empty((max(q.res[2], 0), max(q.res[1], 0), max(q.res[0], 0), 4), dtype=torch.float32, device=torch.device("cuda", self.device))
        s = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        abi.check(self.lib, self.lib.nsb_rgba_on_grid(self.ctx, C.byref(q), d, int(rgb_activation), int(density_activation), out.data_ptr(), s),
                  "nsb_rgba_on_grid")
        return out

    def density_png(self, density, res3d, thresh: float, density_range: float = 4.0, swap_y_z: bool = False, stream=None):
        """save_density_grid_to_png's pixels and counts on a float32 CUDA grid of res3d points (x fastest): (uint8 CUDA tensor [h, w], the
        mosaic of the z slices; int64 CUDA tensor [2]: #zero-x voxels, #lattice near zero-x)."""
        torch = _torch()
        w, h = slices.density_png_extent(res3d, swap_y_z)
        res = (C.c_int32 * 3)(*[int(v) for v in res3d])
        dev = torch.device("cuda", self.device)
        pixels = torch.empty((h, w), dtype=torch.uint8, device=dev)
        counts = torch.empty(2, dtype=torch.int64, device=dev)
        s = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        abi.check(self.lib, self.lib.nsb_density_png(self.ctx, density.data_ptr(), res, float(thresh), float(density_range), int(bool(swap_y_z)),
                                                     pixels.data_ptr(), counts.data_ptr(), s), "nsb_density_png")
        return pixels, counts

    def rgba_png(self, rgba, res3d, swap_y_z: bool = False, stream=None):
        """save_rgba_grid_to_png_sequence's pixels on a float32 CUDA tensor of res3d RGBA points (x fastest): uint8 CUDA tensor
        [slices, h, w, 4], slice z being the image of file %04d_<w>x<h>.png (with the swap: res_y slices of res_z rows)."""
        torch = _torch()
        rx, ry, rz = [int(v) for v in res3d]
        h, n = (rz, ry) if swap_y_z else (ry, rz)
        res = (C.c_int32 * 3)(rx, ry, rz)
        pixels = torch.empty((max(n, 0), max(h, 0), max(rx, 0), 4), dtype=torch.uint8, device=torch.device("cuda", self.device))
        s = torch.cuda.current_stream(self.device).cuda_stream if stream is None else stream
        abi.check(self.lib, self.lib.nsb_rgba_png(self.ctx, rgba.data_ptr(), res, int(bool(swap_y_z)), pixels.data_ptr(), s), "nsb_rgba_png")
        return pixels

