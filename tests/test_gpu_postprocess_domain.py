"""The frame post-process on the GPU over its whole domain, bit for bit against the reference's own CUDA kernels: nsb_accumulate against
accumulate_kernel and nsb_tonemap against tonemap_kernel, both compiled from the reference's render_buffer.cu for sm_90a and launched as
CudaRenderBuffer launches them (16x8 blocks; oracle/ref_video_driver_cuda.cu, refvid_postprocess). Inputs: tests/postprocess_domain.py.

Non-finite values and signed zeros. accumulate_kernel spells fmaxf itself, so the accumulation is compared bit for bit on every input,
NaN equal to NaN. tonemap_kernel clamps with Eigen's cwiseMax / cwiseMin (render_buffer.cu:259, :494). Real Eigen 3.4 evaluates them on
the device as fmaxf / fminf (scalar_max_op / scalar_min_op with PropagateFast -> numext::maxi / mini -> ::fmaxf / ::fminf), which drop
a NaN operand and return +0 for max(-0, +0) on sm_90; k_tonemap uses fmaxf / fminf, so that is what it must compute. The reference's
Eigen is an absent submodule, and the stand-in it is compiled against here spells them a < b ? b : a, which keeps a NaN (and then the
Reinhard luminance spreads it to all three channels) and keeps a -0. So where the two results differ, the difference must be one of
exactly those two, and there the device must compute the documented rule: a -0 of the stand-in is +0, and a NaN of the stand-in is the
value of the CPU oracle's tonemap (fmaxf / fminf, to which nsb_tonemap is pinned) within its powf tolerance. Every other entry,
including every NaN and inf the device produces itself, is compared bit for bit. The tests print how many entries the rule covers.

Where oracle/_ref is absent the reference's stored results (tests/golden/ref/test_gpu_postprocess_domain/) are replayed; large results
keep a seeded sample of whole pixels.
"""
import os

import numpy as np
import pytest

import postprocess_domain as dom
from nerfshop_b200 import abi
from oracle import oracle as orc

pytestmark = pytest.mark.gpu


def _ref_video_available():
    """The reference's post-process kernels can run here (oracle/_ref has a library with refvid_postprocess)."""
    from oracle import ref_video

    return ref_video.serves_postprocess()


_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref", "test_gpu_postprocess_domain")
needs_ref = pytest.mark.skipif(not (_ref_video_available() or os.path.isdir(_GOLDEN)),
                               reason="neither oracle/_ref nor stored reference results (tests/golden/ref/)")


def _same(a, b):
    """Elementwise bit equality, a NaN on both sides counting as equal (the device's NaN payload is canonical)."""
    both = np.isnan(a) & np.isnan(b)
    return both | (a.view(np.uint32) == b.view(np.uint32))


KEEP_PIXELS = 8192  # pixels of a larger frame whose reference results are stored


def _ref_postprocess(frames, spp0, cs, acc0=None, tm_rows=None):
    """ref_video.postprocess through tests/ref_golden.py: (accumulations, surfaces, pixels). A frame of more than KEEP_PIXELS pixels is
    compared whole where oracle/_ref exists, but only a seeded set of its pixels (the first and last among them) is stored and replayed:
    `pixels` names them, or is None for the whole frame."""
    import ref_golden

    from oracle import ref_video

    args = [frames, acc0 if acc0 is not None else np.zeros(0, np.float32), tm_rows if tm_rows is not None else np.zeros(0, np.float32)]
    have = _ref_video_available()
    H, W = (acc0 if acc0 is not None else frames[0]).shape[:2]
    if H * W <= KEEP_PIXELS:
        return ref_golden._call(have, lambda f, a, t: ref_video.postprocess(f, spp0, cs, acc0, tm_rows), *args) + (None,)
    rng = np.random.default_rng(H * W + 7 * spp0 + cs)
    keep = np.unique(np.concatenate([[0, H * W - 1], rng.choice(H * W, KEEP_PIXELS - 2, replace=False)]))
    whole = ref_video.postprocess(frames, spp0, cs, acc0, tm_rows) if have else None
    if whole is not None and not ref_golden.RECORD:
        return whole + (None,)
    kept = ref_golden._call(have, lambda *_: tuple(None if x is None else np.ascontiguousarray(x[keep]) for x in whole), *args, keep)
    return (whole + (None,)) if whole is not None else (kept + (keep,))


def _rows(got, keep):
    return got if keep is None else got[keep]


def _check_tonemap(got, want, oracle_vals, what):
    """got / want / oracle_vals: [pixels, params, 4]. Bit for bit except where the stand-in's clamp differs (module docstring).
    Returns (entries compared, entries under the rule)."""
    same = _same(got, want)
    diff = ~same
    zero_sign = diff & (got == want) & (got == 0)
    nan_kept = diff & np.isnan(want) & ~np.isnan(got)
    other = diff & ~zero_sign & ~nan_kept
    assert not other.any(), (what, int(other.sum()), np.argwhere(other)[:5], got[other][:5], want[other][:5])
    assert not np.signbit(got[zero_sign]).any(), what
    g, o = got[nan_kept], oracle_vals[nan_kept]
    assert np.array_equal(np.isfinite(g), np.isfinite(o)) and np.array_equal(np.isnan(g), np.isnan(o)), what
    fin = np.isfinite(o)
    assert np.allclose(g[fin], o[fin], rtol=1e-5, atol=1e-6), (what, float(np.abs(g[fin] - o[fin]).max()))
    return got.size, int(zero_sign.sum() + nan_kept.sum())


# ---- accumulate ------------------------------------------------------------------------------------------------------------------------
@needs_ref
@pytest.mark.parametrize("shape", list(dom.SHAPES))
def test_accumulate_vs_reference_kernel(renderer, shape):
    """Every colour space, continued sequences from every start index (sample counts around 2^24, where (float)spp + 1 rounds), every
    input class; the accumulation after every call equals accumulate_kernel's, bit for bit."""
    import ref_golden
    import torch

    H, W = dom.SHAPES[shape]
    big = shape == "1920x1080"
    starts, length = (dom.BIG_STARTS, dom.BIG_SEQUENCE) if big else (dom.STARTS, dom.SEQUENCE)
    n_cmp = n_calls = 0
    for ci, (cs_name, cs) in enumerate(dom.COLOR_SPACES.items()):
        for si, start in enumerate(starts):
            seed = 1000 * ci + 10 * si
            frames = np.stack([dom.frame((H, W), seed + 1 + i) for i in range(length)])
            acc0 = dom.frame((H, W), seed) if start else None
            want, _, keep = _ref_postprocess(frames, start, cs, acc0)
            acc = torch.from_numpy(acc0).cuda() if acc0 is not None else torch.full((H, W, 4), np.nan, device="cuda")  # spp 0 clears it
            fr = torch.from_numpy(frames).cuda()
            hist = torch.empty((length, H * W, 4), device="cuda")
            for i in range(length):
                renderer.accumulate(fr[i], acc, start + i, cs)
                hist[i] = acc.reshape(-1, 4)
            got = _rows(hist.permute(1, 0, 2).contiguous().cpu().numpy(), keep)
            got, want = ref_golden.ref.match(got, want)
            bad = ~_same(got, want)
            assert not bad.any(), (cs_name, start, int(bad.sum()), np.argwhere(bad)[:5])
            n_cmp += got.size
            n_calls += length
    print(f"\naccumulate {shape}: {len(dom.COLOR_SPACES) * len(starts)} (colour space x start) sequences of {length}, {n_calls} calls, "
          f"{n_cmp} values bit for bit against accumulate_kernel")


# ---- tonemap -------------------------------------------------------------------------------------------------------------------------------
def _device_tonemap(renderer, acc_t, params):
    import torch

    return torch.stack([renderer.tonemap(acc_t, p).reshape(-1, 4) for p in params], 1).cpu().numpy()


@needs_ref
@pytest.mark.parametrize("cs", list(dom.COLOR_SPACES))
def test_tonemap_vs_reference_kernel(renderer, cs):
    """Input colour space x curve x output space x clamp x exposure x background on the crafted accumulation (every input class):
    nsb_tonemap equals tonemap_kernel bit for bit, non-finite values and signed zeros under the rule of the module docstring."""
    import ref_golden
    import torch

    from oracle import ref_video

    acc = dom.tonemap_input()
    acc_t = torch.from_numpy(acc).cuda()
    px_special = dom.special(acc.reshape(-1, 4))
    total = rule = rule_finite_px = combos = 0
    for curve_name, curve in dom.CURVES.items():
        params = dom.tonemap_params(dom.COLOR_SPACES[cs], curve)
        _, want, _ = _ref_postprocess(np.zeros((0,) + acc.shape, np.float32), 0, dom.COLOR_SPACES[cs], acc, ref_video.tonemap_rows(params))
        got = _device_tonemap(renderer, acc_t, params)
        oracle_vals = np.stack([orc.tonemap(acc, p).reshape(-1, 4) for p in params], 1)
        g, w = ref_golden.ref.match(got, want)
        o, _ = ref_golden.ref.match(oracle_vals, want)
        sp = px_special[want.rows] if isinstance(want, ref_golden.Sampled) else px_special
        n, r = _check_tonemap(g, w, o, (cs, curve_name))
        _, r_fin = _check_tonemap(g[~sp], w[~sp], o[~sp], (cs, curve_name, "finite inputs"))
        total, rule, rule_finite_px, combos = total + n, rule + r, rule_finite_px + r_fin, combos + len(params)
    print(f"\ntonemap {cs}: {combos} parameter sets x {len(dom.CLASSES)} input classes ({len(dom.CLASSES) * combos} combinations), {total} values "
          f"against tonemap_kernel; {total - rule} bit for bit, {rule} under the fmaxf/fminf rule ({rule_finite_px} of them at pixels without "
          f"NaN, inf or -0 inputs: -0 made by the exposure)")


@needs_ref
@pytest.mark.parametrize("shape", list(dom.SHAPES))
def test_tonemap_launch_shapes(renderer, shape):
    """Both launch geometries (256-thread lines on the device, 16x8 blocks in the reference) on every frame shape, every colour space,
    one parameter set per curve."""
    import ref_golden
    import torch

    from oracle import ref_video

    H, W = dom.SHAPES[shape]
    acc = dom.frame((H, W), 77)
    acc_t = torch.from_numpy(acc).cuda()
    settings = ((abi.NSB_TONEMAP_IDENTITY, abi.NSB_COLOR_LINEAR, 0, 0.0, dom.BACKGROUNDS[1]),
                (abi.NSB_TONEMAP_ACES, abi.NSB_COLOR_SRGB, 1, 1.3, dom.BACKGROUNDS[0]),
                (abi.NSB_TONEMAP_HABLE, abi.NSB_COLOR_SRGB, 0, -0.5, dom.BACKGROUNDS[3]),
                (abi.NSB_TONEMAP_REINHARD, abi.NSB_COLOR_LINEAR, 1, 20.0, dom.BACKGROUNDS[4]))
    total = rule = 0
    for cs_name, cs in dom.COLOR_SPACES.items():
        params = []
        for curve, out_cs, clamp, e, bg in settings:
            p = abi.NsbTonemap()
            p.color_space, p.output_color_space, p.tonemap_curve, p.clamp_output_color, p.exposure = cs, out_cs, curve, clamp, e
            p.background_color[:] = bg
            params.append(p)
        _, want, keep = _ref_postprocess(np.zeros((0, H, W, 4), np.float32), 0, cs, acc, ref_video.tonemap_rows(params))
        got = _rows(_device_tonemap(renderer, acc_t, params), keep)
        g, w = ref_golden.ref.match(got, want)
        oracle_vals = _rows(np.stack([orc.tonemap(acc, p).reshape(-1, 4) for p in params], 1), keep)
        o, _ = ref_golden.ref.match(oracle_vals, want)
        n, r = _check_tonemap(g, w, o, (shape, cs_name))
        total, rule = total + n, rule + r
    print(f"\ntonemap {shape}: {total} values against tonemap_kernel, {total - rule} bit for bit, {rule} under the fmaxf/fminf rule")
