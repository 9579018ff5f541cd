"""GPU: every edit-operator entry point over the whole domain of tests/edit_domain.py, bit for bit against the CPU oracle: nsb_map_rays(_op),
nsb_poisson_residuals(_op), nsb_map_positions (stride 3 and 7, with and without a mask, all operators and one at a time),
nsb_poisson_residual_density onto a non-zero fp16 density; the device rebuild of every domain cage after a drag; and one small frame
through k_render_fused<OPS> with the set's operators. NaN results (the flat tet's 0 * inf barycentrics) compare as NaN on both sides."""
import numpy as np
import pytest

import edit_domain as ed
from nerfshop_b200 import abi, editing, synthetic as syn
from oracle import oracle as orc
from test_gpu_edit_rebuild import _check_against_host
from test_gpu_parity import _compare_frames

pytestmark = pytest.mark.gpu


def _same(a, b):
    """Bit equality, a NaN on both sides counting as equal (the device's NaN payload is not the host's)."""
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float32:
        both = np.isnan(a) & np.isnan(b)
        return np.array_equal(np.where(both, 0, a.view(np.uint32)), np.where(both, 0, b.view(np.uint32)))
    return np.array_equal(a, b)


@pytest.fixture()
def ops_restored(renderer):
    yield
    renderer.reset_edit_operators()


def _positions(c, stride):
    p = np.zeros((c.shape[0], stride), np.float32)
    p[:, :3] = c[:, :3]
    p[:, 3:] = np.arange(stride - 3, dtype=np.float32)  # the rest of each row must stay untouched
    return p


@pytest.mark.parametrize("name", ed.NAMES)
def test_entry_points_match_the_oracle(scene, renderer, ops_restored, name):
    import torch

    model, occ = scene
    items = ed.build(model, name)
    ops = ed.ops_of(items)
    o = orc.Oracle(model.desc, model.params, occ, ops)
    renderer.set_edit_operators(ops)
    lib, ctx = renderer.lib, renderer.ctx
    c = ed.samples(model, items)
    n = c.shape[0]

    # map_rays: all operators, then one at a time in reverse list order
    want, want_m = o.map_rays(c)
    assert (want[:, :3] != c[:, :3]).any(1).sum() > 1000
    got, got_m = renderer.map_rays(c)
    assert _same(got, want) and np.array_equal(got_m, want_m)
    ct = torch.from_numpy(c).cuda()
    mask = torch.zeros(n, dtype=torch.uint8, device="cuda")
    for i in range(len(ops) - 1, -1, -1):
        abi.check(lib, lib.nsb_map_rays_op(ctx, i, ct.data_ptr(), mask.data_ptr(), n, None), "map_rays op")
    torch.cuda.synchronize()
    assert _same(ct.cpu().numpy(), want) and np.array_equal(mask.cpu().numpy(), want_m)

    # full membrane residuals, all operators and one at a time
    sh_o, od_o, rd_o = o.poisson_residuals(c)
    sh_g, od_g, rd_g = renderer.poisson_residuals(c)
    assert _same(sh_g, sh_o) and _same(od_g, od_o) and _same(rd_g, rd_o)
    full = [cg.apply_poisson and all(a is not None for a in (cg.boundary_shs, cg.boundary_outside_density, cg.boundary_residual_density)) for cg in ed.cages_of(items)]
    assert ((od_o != 0).sum() > 500) == any(full)
    ct = torch.from_numpy(c).cuda()
    sh, od, rd = torch.zeros((n, 27), device="cuda"), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    for i in range(len(ops) - 1, -1, -1):
        abi.check(lib, lib.nsb_poisson_residuals_op(ctx, i, ct.data_ptr(), n, sh.data_ptr(), od.data_ptr(), rd.data_ptr(), None), "poisson op")
    torch.cuda.synchronize()
    assert _same(sh.cpu().numpy(), sh_o) and _same(od.cpu().numpy(), od_o) and _same(rd.cpu().numpy(), rd_o)

    # map_positions: stride 3 and 7, with and without a mask, all operators (-1) and one at a time
    for stride in (3, 7):
        p0 = _positions(c, stride)
        want_p, want_pm = o.map_positions(p0, np.zeros(n, np.uint8))
        for with_mask in (False, True):
            for per_op in (False, True):
                pt = torch.from_numpy(p0).cuda()
                pm = torch.zeros(n, dtype=torch.uint8, device="cuda")
                mp = pm.data_ptr() if with_mask else None
                for i in (range(len(ops) - 1, -1, -1) if per_op else (-1,)):
                    abi.check(lib, lib.nsb_map_positions(ctx, i, pt.data_ptr(), stride, mp, n, None), "map_positions")
                torch.cuda.synchronize()
                assert _same(pt.cpu().numpy(), want_p), (stride, with_mask, per_op)
                if with_mask:
                    assert np.array_equal(pm.cpu().numpy(), want_pm), (stride, per_op)
    assert _same(want_p[:, :3][~np.isnan(want[:, 0])], want[:, :3][~np.isnan(want[:, 0])])  # positions move as map_rays moves them
    if not any(isinstance(it, editing.CageDeformation) and it.copy for it in items):
        assert np.array_equal(want_pm, want_m)
    else:
        assert (want_pm >= want_m).all() and (want_pm > want_m).any()  # interpolate_tet_pos masks a copy cage's vacated region too

    # residual density onto a non-zero fp16 density, at the mapped positions
    p3 = np.ascontiguousarray(o.map_positions(_positions(c, 3))[0])
    h = np.random.default_rng(7).uniform(-3.0, 20.0, n).astype(np.float16).view(np.uint16)
    want_h = o.poisson_residual_density(p3, h)
    has_rd = [cg.apply_poisson and cg.boundary_residual_density is not None for cg in ed.cages_of(items)]
    assert ((want_h != h).sum() > 500) == any(has_rd)
    for per_op in (False, True):
        pt = torch.from_numpy(p3).cuda()
        ht = torch.from_numpy(h.view(np.int16).copy()).cuda()
        for i in (range(len(ops) - 1, -1, -1) if per_op else (-1,)):
            abi.check(lib, lib.nsb_poisson_residual_density(ctx, i, pt.data_ptr(), 3, ht.data_ptr(), n, None), "residual density")
        torch.cuda.synchronize()
        assert np.array_equal(ht.cpu().numpy().view(np.uint16), want_h), per_op


@pytest.mark.parametrize("name", ed.NAMES)
def test_rebuild_and_frame_match_the_oracle(scene, renderer, ops_restored, name):
    """Drag every domain cage on the device (nsb_cage_deform) and on the host, compare the rebuilt arrays, map the samples again; then one
    small frame with the set's operators through the fused renderer."""
    model, occ = scene
    items = ed.build(model, name)
    renderer.set_edit_operators(ed.ops_of(items))
    dragged = 0
    for i, it in enumerate(items):
        if isinstance(it, editing.CageDeformation):
            renderer.cage_attach_mvc(i, it.mvc)
            moved = it.cage_vertices.copy()
            moved[moved[:, 1] > moved[:, 1].mean()] += np.array([0.03125, -0.0625, 0.015625], np.float32)
            it.cage_vertices = moved
            it.update_tet_mesh()
            renderer.cage_deform(i, moved)
            _check_against_host(renderer, i, it)
            dragged += 1
    assert dragged == len(ed.cages_of(items))
    ops = ed.ops_of(items)
    o = orc.Oracle(model.desc, model.params, occ, ops)
    c = ed.samples(model, items, seed=1, n_random=500)
    want, want_m = o.map_rays(c)
    got, got_m = renderer.map_rays(c)
    assert _same(got, want) and np.array_equal(got_m, want_m)
    target = any(cg.apply_poisson and all(a is not None for a in (cg.boundary_shs, cg.boundary_outside_density, cg.boundary_residual_density))
                 for cg in ed.cages_of(items))
    f = syn.make_frame(model, syn.fox_camera0(), 96, 54, apply_operators=True, poisson_target=target)
    fb_o, depth_o, st_o, margin = o.render(f, want_margin=True)
    fb, depth = renderer.render(f)
    st = renderer.stats()
    _compare_frames(fb.cpu().numpy(), depth.cpu().numpy(), fb_o, depth_o, margin)
    assert abs(int(st.n_samples) - int(st_o.n_samples)) <= max(20, st_o.n_samples // 2000)
    assert st.n_old_samples == st_o.n_old_samples
