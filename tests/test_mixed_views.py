"""Neighbour views of their own width, height and focal length, and 1 to 32
neighbours (SMVSB_MAX_SUBS), against the compiled reference (oracle/_ref) and
the plain restatement (oracle/oracle_port.cc).

Every kernel that reads a neighbour indexes it with that neighbour's own size
and calibration: the bilinear taps of the Gauss-Newton construct, the
z-buffers and 3 % border of the visibility lists, the warp volume and the
consistency check of SGM, the cut of the depth maps, set_scale. The mixed
scene (util_scene.MIXED_SUBS) has a 400x300 main view and neighbours smaller
in both dimensions, portrait, in between, and odd-sized and larger in both
dimensions, at focal lengths 0.85 to 1.3. Tolerances are those of
test_gpu_parity / test_gpu_visibility: 1e-11 on g and H, equal iteration
counts, active sets, lists and cuts, bitwise images and SGM volumes."""
import functools
import os

import numpy as np
import pytest

from oracle import port as oport
from oracle import ref as oref
from smvs_b200 import api, stereo_view, synth

from util_scene import MIXED_SUBS, Pair, make_mixed_scene, rel_err

W, H = 400, 300
needs_ref = pytest.mark.skipif(not oref.available(), reason="oracle/_ref not built")
needs_port = pytest.mark.skipif(not oport.available(), reason="oracle port not built")
TOL = 1e-11


@functools.lru_cache(maxsize=None)
def mixed_scene(shading=False, init_noise=0.02):
    """Read-only: shared by the tests of this file. At the default 2 % depth
    noise a Newton loop from the initial surface stops after one step; the
    loop tests start from 10 % (5 steps on the mixed scene)."""
    return make_mixed_scene(W, H, MIXED_SUBS, seed_index=80, shading=shading,
                            init_noise=init_noise)


@functools.lru_cache(maxsize=None)
def uniform_scene(n_sub, w=160, h=120):
    """n_sub neighbours of the main view's size, for the neighbour counts."""
    return make_mixed_scene(w, h, [(w, h, 1.0)] * n_sub, seed_index=81 + n_sub,
                            init_noise=0.1)


def projections(Mi, ti, k, depth, ps=1):
    """Main-view pixel centres (every ps-th pixel) at `depth` projected into
    neighbour k as the construct kernel does it (Correspondence::fill and the
    caller's -0.5): (x, y) in the neighbour's pixel coordinates."""
    h, w = depth.shape
    ys, xs = np.mgrid[0:h:ps, 0:w:ps]
    u, v = xs + 0.5, ys + 0.5
    d = depth[::ps, ::ps].astype(np.float64)
    M = Mi[k].reshape(3, 3)
    p = [M[i, 0] * u + M[i, 1] * v + M[i, 2] for i in range(3)]
    a, b, c = (d * p[i] + ti[k][i] for i in range(3))
    return a / c - 0.5, b / c - 0.5


def lists_of(off, ids, valid):
    return [tuple(ids[off[p]:off[p + 1]]) if valid[p] else () for p in range(len(valid))]


def listed_fraction(off, ids, pv, k):
    lists = [l for l in lists_of(off, ids, pv) if l]
    return float(np.mean([k in l for l in lists]))


# ---------------------------------------------------------------------------
# CPU: the checker and the scene
# ---------------------------------------------------------------------------

@needs_ref
@pytest.mark.parametrize("scale", [0, 2, 4])
def test_ref_scene_returns_each_views_own_shape(scale):
    """RefScene's per-view accessors allocate the view's own shape. The
    417x311 neighbour is larger than the main view: a buffer of the main
    view's shape would be overrun. Each image is bitwise the numpy set_scale
    mirror (pinned to the reference by test_cpu_host) of that view alone."""
    sc = mixed_scene()
    R = oref.RefScene(sc)
    try:
        R.set_scale(scale)
        for v in range(1 + sc.n_sub):
            shape = sc.images[v].shape
            g, hs, blur = R.gradients(v), R.hessian(v), R.scaleimage(v)
            assert g.shape == shape + (2,) and hs.shape == shape + (3,)
            assert blur.shape == shape
            rb, rg, rh = stereo_view.set_scale(sc.images[v], scale)
            assert np.array_equal(blur, rb), v
            assert np.array_equal(g, rg), v
            assert np.array_equal(hs, rh), v
    finally:
        R.close()


@needs_ref
def test_mixed_scene_exercises_what_it_claims():
    """The scene is not vacuous: every neighbour is listed for a good share
    of the patches, the portrait and the smallest neighbour see main-view
    samples fall outside their image (the clamps of the bilinear taps run),
    the u8 widths take both set_scale paths, and the reprojections are not
    those of an equal-size scene."""
    sc = mixed_scene()
    assert [im.shape[::-1] for im in sc.images[1:]] == [s[:2] for s in MIXED_SUBS]
    assert np.array_equal(sc.flen[1:], np.float32([s[2] for s in MIXED_SUBS]))
    widths = [im.shape[1] for im in sc.images]
    assert {w % 16 == 0 for w in widths} == {True, False}      # TMA and three kernels
    big = sc.images[4].shape
    assert big[0] > H and big[1] > W and big[0] % 2 == 1 and big[1] % 2 == 1
    R = oref.RefScene(sc)
    try:
        R.set_scale(2)
        R.surface_create(2, sc.init_depth)
        R.compute_visibility()
        _, _, pv = R.surface_get()
        off, ids = R.get_visibility()
        # measured with the compiled reference: 0.51, 0.70, 0.69, 1.00
        for k in range(sc.n_sub):
            assert listed_fraction(off, ids, pv, k) > 0.4, k
        Mi, ti = R.Mt()
        for k in (0, 1):
            w, h = MIXED_SUBS[k][:2]
            x, y = projections(Mi, ti, k, sc.true_depth)
            out = (x < 0) | (x > w - 1) | (y < 0) | (y > h - 1)
            assert 0.1 < out.mean() < 0.6, (k, out.mean())   # 0.43, 0.25
        # Mi = K_k R_k K_0^-1 with the neighbour's own calibration
        K0inv = np.linalg.inv(synth.calibration(1.0, W, H))
        eq = make_mixed_scene(W, H, [(W, H, 1.0)] * sc.n_sub, seed_index=80)
        Re = oref.RefScene(eq)
        Mie, tie = Re.Mt()
        Re.close()
        for k, (w, h, f) in enumerate(MIXED_SUBS):
            K = synth.calibration(float(np.float32(f)), w, h)
            M = K @ sc.rot[k + 1].astype(np.float64).reshape(3, 3) @ K0inv
            assert rel_err(Mi[k], M.reshape(9)) < 1e-6
            assert rel_err(ti[k], K @ sc.trans[k + 1].astype(np.float64)) < 1e-6
            assert rel_err(Mi[k], Mie[k]) > 1e-2 and rel_err(ti[k], tie[k]) > 1e-3
    finally:
        R.close()


def _port_of(R, n_sub):
    Mi, ti = R.Mt()
    return oport.PortScene(R.gradients(0), [R.gradients(k + 1) for k in range(n_sub)],
                           [R.hessian(k + 1) for k in range(n_sub)], Mi, ti, R.flen(0),
                           R.inverse_flen(0))


@needs_ref
@needs_port
@pytest.mark.parametrize("case", ["mixed", "n32"])
def test_port_construct_and_cg_match_the_reference(case):
    """The restatement is the checker a build without the reference uses:
    it must hold at per-view sizes and at 32 neighbours (496 pair rows per
    sample)."""
    sc = mixed_scene() if case == "mixed" else uniform_scene(32)
    R = oref.RefScene(sc)
    try:
        R.set_scale(2)
        R.surface_create(2, sc.init_depth)
        R.compute_visibility()
        info = R.surface_info()
        nodes, nv, pv = R.surface_get()
        off, ids = R.get_visibility()
        lens = np.diff(off.astype(np.int64))[pv.astype(bool)]
        assert lens.max() == sc.n_sub
        P = _port_of(R, sc.n_sub)
        P.set_surface(info["scale"], info["npx"], info["npy"], info["start_x"],
                      info["start_y"], nodes, nv, pv, off, ids)
        R.gn_construct(nv, None, 0.01, 0.0)
        P.gn_construct(nv, None, 0.01, 0.0)
        rs, ps = R.get_system(), P.get_system()
        for k in ("Houter", "Hinner", "Pouter", "Pinner"):
            assert np.array_equal(ps[k], rs[k]), k
        assert rel_err(ps["g"], rs["g"]) < TOL
        assert rel_err(ps["Hvals"], rs["Hvals"]) < TOL
        xr, itr, infr = R.cg_solve()
        xp, itp, infp = P.cg_solve()
        assert (itp, infp) == (itr, infr)
        assert rel_err(xp, xr) < 1e-6
        P.close()
    finally:
        R.close()


def occluded_mixed_scene(sc):
    """occluded_scene of test_gpu_visibility on a given scene: a raised block
    in the initial depth, a foreground disc and holes in the SGM depth."""
    init = sc.init_depth.copy()
    init[H // 3:H // 2, W // 3:W // 2] *= 0.8
    yy, xx = np.mgrid[0:H, 0:W]
    sgm = sc.init_depth.copy()
    sgm[(xx - 0.7 * W) ** 2 + (yy - 0.6 * H) ** 2 < (0.12 * H) ** 2] *= 0.6
    sgm[(xx + 2 * yy) % 17 == 0] = 0.0
    return init.astype(np.float32), sgm.astype(np.float32)


@needs_ref
@needs_port
def test_port_visibility_and_cutting_match_the_reference():
    sc = mixed_scene()
    init, sgm = occluded_mixed_scene(sc)
    R = oref.RefScene(sc)
    try:
        R.set_scale(3)
        R.surface_create(3, init)
        R.set_sgm_depth(sgm)
        info = R.surface_info()
        nodes, nv, pv = R.surface_get()
        P = _port_of(R, sc.n_sub)
        P.set_surface(info["scale"], info["npx"], info["npy"], info["start_x"],
                      info["start_y"], nodes, nv, pv, None, None)
        left = R.create_subview_surfaces(True)
        removed = P.visibility(sgm)
        assert int(pv.sum()) - removed == left and removed > 0
        _, nv_r, pv_r = R.surface_get()
        off_r, ids_r = R.get_visibility()
        nv_p, pv_p, off_p, ids_p = P.surface_state()
        assert np.array_equal(pv_p, pv_r) and np.array_equal(nv_p, nv_r)
        assert lists_of(off_p, ids_p, pv_p) == lists_of(off_r, ids_r, pv_r)
        K = R.inverse_calibration()
        cuts = []
        for _ in range(12):
            d = R.cut_boundaries()
            assert P.cut_boundaries(K) == d
            _, nv_r, pv_r = R.surface_get()
            nv_p, pv_p, _, _ = P.surface_state()
            assert np.array_equal(pv_p, pv_r) and np.array_equal(nv_p, nv_r)
            cuts.append(d)
            if d <= 10:
                break
        assert sum(cuts) > 0
        P.close()
    finally:
        R.close()


# SGM at an odd main size with neighbours larger, smaller and portrait
SGM_W, SGM_H = 333, 207
SGM_SUBS = ((417, 311, 0.85), (256, 192, 1.3), (207, 333, 1.0))


@functools.lru_cache(maxsize=None)
def sgm_scene():
    sc = make_mixed_scene(SGM_W, SGM_H, SGM_SUBS, seed_index=82)
    dmin, dmax = float(sc.true_depth.min() * 0.7), float(sc.true_depth.max() * 1.3)
    return sc, dmin, dmax


@needs_ref
@needs_port
@pytest.mark.parametrize("k", [1, 2, 3])
def test_port_sgm_with_other_neighbour_size(k):
    sc, dmin, dmax = sgm_scene()
    nh, nw = sc.images[k].shape
    assert (nw, nh) != (SGM_W, SGM_H)
    R = oref.RefScene(sc)
    r = R.sgm_run(0, k, 0, 64, dmin, dmax, volumes=True)
    M, t = R.reprojection(0, k, SGM_W, SGM_H, nw, nh)
    R.close()
    p = oport.sgm(sc.images[0], sc.images[k], M, t, dmin, dmax, 64)
    assert np.array_equal(p["cost"], r["cost"])
    assert np.array_equal(p["sgm"], r["sgm"])
    assert np.array_equal(p["depth"], r["depth"])
    assert (r["depth"] > 0).mean() > 0.2


# ---------------------------------------------------------------------------
# GPU against the compiled reference
# ---------------------------------------------------------------------------

@pytest.mark.gpu
@needs_ref
def test_set_views_u8_per_view_sizes():
    """smvsb_set_views_u8 runs set_scale on each neighbour at its own size
    through staging buffers sized by the largest view; widths 400, 256, 352
    take the TMA kernel, 300 and 417 the three kernels."""
    sc = mixed_scene()
    R = oref.RefScene(sc)
    Mi, ti = R.Mt()
    try:
        with api.Context(0) as ctx:
            for scale in (1, 2, 4):
                R.set_scale(scale)
                ctx.set_views_u8(scale, sc.images[0], sc.images[1:], Mi, ti, R.flen(0),
                                 R.inverse_flen(0))
                g, _ = ctx.debug_get_view(0)
                assert np.array_equal(g, R.gradients(0)), scale
                for k in range(1, 1 + sc.n_sub):
                    g, hs = ctx.debug_get_view(k)
                    assert g.shape[:2] == sc.images[k].shape
                    assert np.array_equal(g, R.gradients(k)), (scale, k)
                    assert np.array_equal(hs, R.hessian(k)), (scale, k)
    finally:
        R.close()


def _restrict_to(P, keep):
    """Lists cut down to the neighbours in `keep`; patches left without one
    are removed with the nodes only they held (the same surface on both
    sides)."""
    npx, npy = P.info["npx"], P.info["npy"]
    off, ids = [0], []
    pv = P.patch_valid0.copy()
    for p in range(npx * npy):
        lst = [int(i) for i in P.vis_ids0[P.vis_off0[p]:P.vis_off0[p + 1]] if int(i) in keep]
        if not lst:
            pv[p] = 0
        ids += lst
        off.append(len(ids))
    nv = np.zeros_like(P.node_valid0)
    pv2, nv2 = pv.reshape(npy, npx), nv.reshape(npy + 1, npx + 1)
    for dy in (0, 1):
        for dx in (0, 1):
            nv2[dy:dy + npy, dx:dx + npx] |= pv2
    nv &= P.node_valid0
    P.node_valid, P.patch_valid = nv, pv
    P.vis_off, P.vis_ids = np.array(off, np.uint32), np.array(ids, np.uint8)
    P.R.surface_set(P.nodes, nv, pv)
    P.R.set_visibility(P.vis_off, P.vis_ids)
    P.push_surface()
    return int(pv.sum())


def _all_listed(P):
    """Every neighbour listed for every valid patch: samples fall outside the
    smaller neighbours, the clamps of the bilinear taps run."""
    n, npatch = P.scene.n_sub, len(P.patch_valid0)
    P.vis_off0 = np.arange(npatch + 1, dtype=np.uint32) * n
    P.vis_ids0 = np.tile(np.arange(n, dtype=np.uint8), npatch)


def _construct_solve_update(P, light=None):
    from test_gpu_parity import assert_system_equal
    act = P.node_valid
    P.R.gn_construct(act, light, 0.01, 0.0)
    P.ctx.gn_construct(act, light, 0.01, 0.0)
    assert_system_equal(P.ctx.debug_get_system(), P.R.get_system())
    xr, itr, infr = P.R.cg_solve()
    itg, infg = P.ctx.cg_solve()
    assert (itg, infg) == (itr, infr)
    if itr < 200:
        assert rel_err(P.ctx.get_delta(), xr) < 1e-8
    else:
        # stopped by max_iterations: rounding differences of 1e-14 in H are
        # amplified by the unconverged Krylov process in any implementation
        # (test_full_size_live_parity); the update runs on the reference's x
        assert infr == 1 and rel_err(P.ctx.get_delta(), xr) < 1e-3
        P.ctx.set_delta(xr)
    ar, nr, _ = P.R.update_nodes(xr, act)
    ag, ng, _ = P.ctx.update_nodes()
    assert ng == nr and np.array_equal(ag, ar)
    P.R.surface_set(P.nodes, P.node_valid, P.patch_valid)
    P.push_surface()


def _mixed_pair(scale, shading, init_noise=0.02):
    sc = mixed_scene(shading, init_noise)
    P = Pair(W, H, sc.n_sub, scale, shading=shading, scene=sc)
    P.vis_off0, P.vis_ids0 = P.vis_off, P.vis_ids
    P.patch_valid0, P.node_valid0 = P.patch_valid.copy(), P.node_valid.copy()
    return P


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("scale,shading", [(2, False), (3, False), (1, False), (2, True)])
def test_construct_cg_update_per_neighbour(scale, shading):
    """Construct, PCG and update on the mixed scene: once with the lists of
    compute_visibility, once with every neighbour listed everywhere (the
    clamps run), then once per neighbour with the lists cut down to it, so
    that a fault in one neighbour's addressing is the whole system and cannot
    hide under the max-relative error of the others."""
    P = _mixed_pair(scale, shading)
    try:
        light = P.R.fit_lighting() if shading else None
        if shading:
            assert rel_err(P.ctx.fit_lighting(), light) < 1e-5
        n = P.scene.n_sub
        lens = np.diff(P.vis_off0.astype(np.int64))[P.patch_valid0.astype(bool)]
        assert lens.max() == n and lens.min() >= 1
        _construct_solve_update(P, light)
        for k in range(n):
            left = _restrict_to(P, {k})
            assert left > 0.3 * int(P.patch_valid0.sum()), (k, left)
            _construct_solve_update(P, light)
        _all_listed(P)
        # some samples of the smallest and the portrait neighbour lie outside them
        Mi, ti = P.Mi, P.ti
        for k in (0, 1):
            w, h = MIXED_SUBS[k][:2]
            x, y = projections(Mi, ti, k, P.scene.init_depth, 1 << max(scale, 1))
            assert ((x < 0) | (x > w - 1) | (y < 0) | (y > h - 1)).mean() > 0.1
        for keep in (set(range(n)), {0}, {1}):
            assert _restrict_to(P, keep) == int(P.patch_valid0.sum())
            _construct_solve_update(P, light)
    finally:
        P.close()


def _loop_parity(P, light=None):
    sr = P.R.newton_loop(light, 0.01, 0.0)
    sg = P.ctx.newton_loop(light, 0.01, 0.0)
    for k in ("newton_steps", "cg_iterations", "n_active", "pixel_iterations"):
        assert sg[k] == sr[k], k
    assert sr["newton_steps"] > 1
    d, dr = P.ctx.get_depth(), P.R.surface_depth()
    assert np.array_equal(d > 0, dr > 0) and rel_err(d, dr) < 1e-6
    return sg


@pytest.mark.gpu
@needs_ref
def test_newton_loop_mixed_scene():
    P = _mixed_pair(2, False, init_noise=0.1)
    try:
        _loop_parity(P)
    finally:
        P.close()


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("n_sub", [1, 7, 32])
def test_neighbour_counts(n_sub):
    """1 neighbour (no pair rows), 7 and 32 (SMVSB_MAX_SUBS, 496 pair rows
    per sample): visibility lists of full length, construct, PCG, update and
    the whole Newton loop."""
    sc = uniform_scene(n_sub)
    P = Pair(160, 120, n_sub, 2, scene=sc)
    try:
        lens = np.diff(P.vis_off.astype(np.int64))[P.patch_valid.astype(bool)]
        assert lens.max() == n_sub
        if n_sub == 32:
            assert (lens == 32).mean() > 0.3
        # the device's own lists from the same surface: equal
        with api.Context(0) as ctx:
            ctx.set_views(P.R.gradients(0), [P.R.gradients(k + 1) for k in range(n_sub)],
                          [P.R.hessian(k + 1) for k in range(n_sub)], P.Mi, P.ti,
                          P.R.flen(0), P.R.inverse_flen(0))
            R2 = oref.RefScene(sc)
            R2.set_scale(2)
            R2.surface_create(2, sc.init_depth)
            R2.set_sgm_depth(sc.init_depth)
            info = R2.surface_info()
            nodes, nv, pv = R2.surface_get()
            ctx.set_surface(info["scale"], info["npx"], info["npy"], info["start_x"],
                            info["start_y"], nodes, nv, pv, None, None)
            left = R2.create_subview_surfaces(True)
            ctx.visibility(sc.init_depth)
            _, nv_r, pv_r = R2.surface_get()
            off_r, ids_r = R2.get_visibility()
            nv_g, pv_g, off_g, ids_g = ctx.surface_state()
            R2.close()
            assert int(pv_g.sum()) == left
            assert np.array_equal(pv_g, pv_r) and np.array_equal(nv_g, nv_r)
            lr = lists_of(off_r, ids_r, pv_r)
            assert lists_of(off_g, ids_g, pv_g) == lr
            assert max(len(l) for l in lr) == n_sub
        P.vis_off0, P.vis_ids0 = P.vis_off, P.vis_ids
        P.patch_valid0, P.node_valid0 = P.patch_valid.copy(), P.node_valid.copy()
        _construct_solve_update(P)
        _loop_parity(P)
    finally:
        P.close()


@pytest.mark.gpu
def test_more_than_32_neighbours_is_rejected():
    n = 33
    g2, g3 = np.zeros((16, 16, 2), np.float32), np.zeros((16, 16, 3), np.float32)
    img = np.zeros((16, 16), np.uint8)
    Mi, ti = np.tile(np.eye(3).reshape(9), (n, 1)), np.zeros((n, 3))
    with api.Context(0) as ctx:
        last = lambda: api.lib().smvsb_last_error(ctx._h)  # noqa: E731
        with pytest.raises(api.SmvsbError) as e:
            ctx.set_views(g2, [g2] * n, [g3] * n, Mi, ti, 16.0, 1.0 / 16.0)
        assert e.value.code == -1 and b"n_sub" in last()
        with pytest.raises(api.SmvsbError) as e:
            ctx.set_views_u8(2, img, [img] * n, Mi, ti, 16.0, 1.0 / 16.0)
        assert e.value.code == -1 and b"n_sub" in last()
        with pytest.raises(api.SmvsbError) as e:
            api.optimize(ctx, img, [img] * n, Mi, ti, 16.0, 1.0 / 16.0,
                         np.eye(3, dtype=np.float32), np.ones((16, 16), np.float32))
        assert e.value.code == -1 and b"neighbour" in last()
        # 32 is accepted
        ctx.set_views(g2, [g2] * 32, [g3] * 32, Mi[:32], ti[:32], 16.0, 1.0 / 16.0)


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("use_sgm,scale", [(True, 2), (True, 3), (False, 3)])
def test_visibility_and_cut_mixed(use_sgm, scale):
    """Deleted patches, nodes, lists and cut counts EQUAL to the reference's;
    use_sgm = false reads the colour images at their own sizes."""
    sc = mixed_scene()
    if not use_sgm:     # the recipe of util_scene.colour_scene, per view
        import copy
        col = copy.copy(sc)
        rng = np.random.default_rng(83)
        col.images = [np.stack([np.clip(im.astype(np.float32) * g + o
                                        + rng.normal(0, 2.0, im.shape), 0, 255)
                                for g, o in ((1.0, 0.0), (0.8, 20.0), (1.1, -10.0))],
                               axis=2).astype(np.uint8) for im in sc.images]
        sc = col
    init, sgm = occluded_mixed_scene(sc)
    R = oref.RefScene(sc)
    n = sc.n_sub
    try:
        R.set_scale(scale)
        R.surface_create(scale, init)
        if use_sgm:
            R.set_sgm_depth(sgm)
        info = R.surface_info()
        nodes, nv, pv = R.surface_get()
        Mi, ti = R.Mt()
        with api.Context(0) as ctx:
            ctx.set_views(R.gradients(0), [R.gradients(k + 1) for k in range(n)],
                          [R.hessian(k + 1) for k in range(n)], Mi, ti,
                          R.flen(0), R.inverse_flen(0))
            ctx.set_surface(info["scale"], info["npx"], info["npy"], info["start_x"],
                            info["start_y"], nodes, nv, pv, None, None)
            assert np.array_equal(ctx.get_depth(), R.surface_depth())
            if not use_sgm:
                imgs = [R.image(v) for v in range(1 + n)]
                assert [im.shape[:2] for im in imgs] == [im.shape[:2] for im in sc.images]
                ctx.set_color_images(imgs[0], imgs[1:])
            left = R.create_subview_surfaces(use_sgm)
            removed = ctx.visibility(sgm if use_sgm else None)
            _, nv_r, pv_r = R.surface_get()
            off_r, ids_r = R.get_visibility()
            nv_g, pv_g, off_g, ids_g = ctx.surface_state()
            assert np.array_equal(pv_g, pv_r) and np.array_equal(nv_g, nv_r)
            assert int(pv.sum()) - removed == left == int(pv_g.sum())
            lr = lists_of(off_r, ids_r, pv_r)
            assert lists_of(off_g, ids_g, pv_g) == lr
            # every neighbour listed somewhere, some lists partial
            assert all(any(k in l for l in lr) for k in range(n))
            assert any(0 < len(l) < n for l in lr)
            K = R.inverse_calibration()
            total = 0
            for _ in range(12):
                d_r, d_g = R.cut_boundaries(), ctx.cut_boundaries(K)
                _, nv_r, pv_r = R.surface_get()
                nv_g, pv_g, _, _ = ctx.surface_state()
                assert d_g == d_r
                assert np.array_equal(pv_g, pv_r) and np.array_equal(nv_g, nv_r)
                total += d_r
                if d_r <= 10:
                    break
            if use_sgm:
                assert removed > 0 and total > 0
    finally:
        R.close()


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("k", [1, 2, 3])
@pytest.mark.parametrize("D", [64, 128])
def test_sgm_neighbour_of_other_size(k, D):
    """Cost, aggregated volume and depth bit-exact with the neighbour at its
    own size; the 333x207 main view gives the 128-plane kernels odd line
    counts in every direction."""
    sc, dmin, dmax = sgm_scene()
    assert SGM_W % 2 == 1 and SGM_H % 2 == 1
    nh, nw = sc.images[k].shape
    R = oref.RefScene(sc)
    r = R.sgm_run(0, k, 0, D, dmin, dmax, volumes=True)
    M, t = R.reprojection(0, k, SGM_W, SGM_H, nw, nh)
    R.close()
    g = api.sgm(sc.images[0], sc.images[k], M, t, dmin, dmax, D, volumes=True)
    assert np.array_equal(g["cost"], r["cost"])
    assert np.array_equal(g["sgm"], r["sgm"])
    assert np.array_equal(g["depth"], r["depth"])
    assert (r["depth"] > 0).mean() > 0.2


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("p1,p2", [(6, 96), (96, 96), (1, 255), (255, 255)])
def test_sgm_penalties(p1, p2):
    """Penalties up to check_sgm_args' limit: the byte volumes rely on
    L - C <= P2 <= 255. The reference runs each pair first."""
    sc, dmin, dmax = sgm_scene()
    nh, nw = sc.images[1].shape
    R = oref.RefScene(sc)
    M, t = R.reprojection(0, 1, SGM_W, SGM_H, nw, nh)
    for D in (64, 128):
        r = R.sgm_run(0, 1, 0, D, dmin, dmax, p1, p2, volumes=True)
        assert (r["depth"] > 0).any() and r["sgm"].max() > 0
        g = api.sgm(sc.images[0], sc.images[1], M, t, dmin, dmax, D, p1, p2, volumes=True)
        assert np.array_equal(g["cost"], r["cost"]), D
        assert np.array_equal(g["sgm"], r["sgm"]), D
        assert np.array_equal(g["depth"], r["depth"]), D
    R.close()


@pytest.mark.gpu
@needs_ref
def test_sgm_reconstruct_neighbours_of_other_sizes():
    """smvsb_sgm_reconstruct with nw x nh != w x h: the larger neighbour first
    (the workspace grows between the two runs of one call), then the smaller
    and the portrait one merged in, against SGMStereo::reconstruct and the
    merge of app/smvsrecon.cc:362-377."""
    sc, dmin, dmax = sgm_scene()
    R = oref.RefScene(sc)
    order = (1, 2, 3)
    ref = {k: R.sgm_reconstruct(0, k, 0, 64, dmin, dmax) for k in order}
    prev, merged = None, None
    for k in order:
        nh, nw = sc.images[k].shape
        M_mn, t_mn = R.reprojection(0, k, SGM_W, SGM_H, nw, nh)
        M_nm, t_nm = R.reprojection(k, 0, nw, nh, SGM_W, SGM_H)
        args = (sc.images[0], sc.images[k], M_mn, t_mn, M_nm, t_nm, (dmin, dmax),
                (dmin, dmax), 64)
        single = api.sgm_reconstruct(*args)["depth"]
        assert np.array_equal(single, ref[k]), k
        assert 0.1 < (single > 0).mean() < 1.0, k
        prev = api.sgm_reconstruct(*args, merge_with=prev)["depth"]
        if merged is None:
            merged = ref[k].copy()
        else:
            d2 = ref[k]
            both = (merged != 0) & (d2 != 0)
            only2 = (merged == 0) & (d2 != 0)
            merged[both] = (merged[both] + d2[both]) * np.float32(0.5)
            merged[only2] = d2[only2]
        assert np.array_equal(prev, merged), k
    R.close()


@pytest.mark.gpu
@needs_ref
def test_cut_depth_maps_views_of_other_sizes():
    from test_gpu_cutmaps import make_views
    sizes = [(320, 240, 1.1), (256, 192, 1.3), (240, 320, 1.0), (353, 263, 0.9)]
    flen, rot, trans, depths, normals = make_views(len(sizes), 0, 0, 7, sizes=sizes)
    outs, inv, ctw, KR, t = oref.cut_depth_maps(flen, rot, trans, depths, normals)
    got = api.cut_depth_maps(depths, normals, inv, ctw, KR, t)
    for k, (g, o, d) in enumerate(zip(got, outs, depths)):
        assert g.shape == d.shape == sizes[k][1::-1]
        assert np.array_equal(g, o), k
        assert (o > 0).mean() > 0.1 and ((o == 0) & (d > 0)).mean() > 0.02, k


@pytest.mark.gpu
@needs_ref
def test_resident_optimize_mixed_scene():
    """smvsb_optimize with neighbours of their own sizes against the
    reference's DepthOptimizer::optimize(), as in
    test_resident_optimize_matches_reference."""
    sc = mixed_scene()
    R = oref.RefScene(sc)
    d_cpu, n_cpu, _ = R.optimize(sc.init_depth, regularization=0.01, num_iterations=5,
                                 min_scale=2)
    Mi, ti = R.Mt()
    sgm = R.sgm_roundtrip(sc.init_depth)
    with api.Context(0) as ctx:
        d, n, _, st = api.optimize(ctx, sc.images[0], sc.images[1:], Mi, ti, R.flen(0),
                                   R.inverse_flen(0), R.inverse_calibration(), sgm)
    R.close()
    assert st["final_scale"] == 2 and st["newton_steps"] > 5
    assert np.array_equal(d_cpu > 0, d > 0)
    m = d_cpu > 0
    assert m.mean() > 0.5
    assert (np.abs(d[m] - d_cpu[m]) / d_cpu[m]).max() < 1e-6
    assert np.abs(n - n_cpu)[m].max() < 1e-5


@pytest.mark.gpu
@pytest.mark.skipif(not (oref.available() and os.path.exists(oref.INTEGRATION_LIB_PATH)),
                    reason="oracle/_ref or oracle/_ref/integration not built")
def test_drop_in_optimize_mixed_scene(monkeypatch):
    """The reference's optimize() through the drop-in build against the
    pure-CPU build on the mixed scene (tolerances of test_integration)."""
    monkeypatch.delenv("SMVSB_MEMBERWISE", raising=False)
    sc = mixed_scene()
    out = []
    for path in (None, oref.INTEGRATION_LIB_PATH):
        R = oref.RefScene(sc, lib_path=path)
        before = api.lib().smvsb_global_launch_count()
        d, n, _ = R.optimize(sc.init_depth, regularization=0.01, num_iterations=5,
                             min_scale=2)
        assert (api.lib().smvsb_global_launch_count() - before > 20) == (path is not None)
        R.close()
        out.append((d, n))
    (d_cpu, n_cpu), (d_gpu, n_gpu) = out
    assert np.array_equal(d_cpu > 0, d_gpu > 0)
    m = d_cpu > 0
    assert m.mean() > 0.5
    assert (np.abs(d_gpu[m] - d_cpu[m]) / d_cpu[m]).max() < 1e-4
    assert np.abs(n_gpu - n_cpu).max() < 1e-3


@pytest.mark.gpu
@needs_ref
def test_batch_with_mixed_scene_is_the_single_loop():
    """smvsb_newton_loop_batch over the mixed scene and a uniform one: each
    view bitwise its own single loop."""
    pairs = [_mixed_pair(2, False, init_noise=0.1),
             Pair(160, 120, 7, 2, scene=uniform_scene(7))]
    try:
        ctxs = [p.ctx for p in pairs]
        single, nodes = [], []
        for p in pairs:
            single.append(p.ctx.newton_loop(None, 0.01, 0.0))
            nodes.append(p.ctx.get_nodes())
            p.ctx.set_nodes(p.nodes)
        batch = api.newton_loop_batch(ctxs, None, 0.01, 0.0)
        for k, (p, s, b) in enumerate(zip(pairs, single, batch)):
            for key in ("newton_steps", "cg_iterations", "n_active", "pixel_iterations",
                        "nan", "cg_block_iterations", "cg_row_iterations"):
                assert b[key] == s[key], (k, key)
            assert np.array_equal(p.ctx.get_nodes(), nodes[k]), k
    finally:
        for p in pairs:
            p.close()
