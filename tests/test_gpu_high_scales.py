"""Surfaces whose coarse-to-fine ladder starts at scale 7 or 8 (patch size 128
or 256, 1024 or 4096 Gauss-Newton samples per patch): what optimize() starts
at for photographs of about 7 MP and more without SGM and 27 MP and more with
it. Every stage against the compiled reference (oracle/_ref) on small images
first -- set_scale, surface creation and subdivision, the Gauss-Newton
system, a Newton loop, visibility in both modes and boundary cutting -- then
the whole resident optimize() from scale 7 and from scale 8, and the drop-in
optimize() from scale 7."""
import os
import subprocess
import sys

import numpy as np
import pytest

from smvs_b200 import api, synth
from oracle import ref as oref

from test_gpu_parity import assert_system_equal
from test_gpu_topology import _features_on_surface
from util_scene import Pair, colour_scene, rel_err

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
import highres_cpu as hc  # noqa: E402

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not oref.available(), reason="oracle/_ref not built")]


@pytest.fixture(scope="module", autouse=True)
def ladder8_reference():
    """The CPU reference of the scale-8 ladder (about 12 minutes on one host
    core): from benchmarks/_cache/ when present, otherwise computed by
    benchmarks/highres_cpu.py in a subprocess started with the module's first
    test, so that it runs while the other tests do."""
    proc = None
    if not os.path.exists(hc.cache_path()):
        proc = subprocess.Popen([sys.executable, os.path.join(ROOT, "benchmarks", "highres_cpu.py")],
                                stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)

    def get():
        nonlocal proc
        if proc is not None:
            out, _ = proc.communicate(timeout=1800)
            assert proc.returncode == 0, out[-2000:]
            proc = None
        return np.load(hc.cache_path())

    yield get
    if proc is not None:
        proc.kill()
        proc.wait()


# 9 x 7 patches at scale 7, 4 x 3 at scale 8
W, H = 1300, 1060


def _lists(off, ids, valid):
    return [tuple(ids[off[p]:off[p + 1]]) if valid[p] else () for p in range(len(valid))]


def _ctx_with_sizes(R, n_sub, w=W, h=H):
    """A context that knows the view sizes and poses (the surface operations
    read no image data)."""
    ctx = api.Context(0)
    Mi, ti = R.Mt()
    z2, z3 = np.zeros((h, w, 2), np.float32), np.zeros((h, w, 3), np.float32)
    ctx.set_views(z2, [z2] * n_sub, [z3] * n_sub, Mi, ti, R.flen(0), R.inverse_flen(0))
    return ctx


def _assert_surface_equal(ctx, R, what):
    assert ctx.surface_info() == R.surface_info(), what
    nodes = ctx.get_nodes()
    nv, pv, _, _ = ctx.surface_state()
    rn, rnv, rpv = R.surface_get()
    assert np.array_equal(nv, rnv), what
    assert np.array_equal(pv, rpv), what
    assert np.array_equal(nodes[rnv.astype(bool)], rn[rnv.astype(bool)]), what


def _init_depth(sc, seed):
    """The scene's initial depth with holes and, over a quarter of the image,
    depths rounded to a few values: node windows there hold thousands of
    equal depths, so the median must follow std::nth_element's tie rule."""
    rng = np.random.default_rng(seed)
    d = sc.init_depth.astype(np.float32).copy()
    h, w = d.shape
    d[rng.random(d.shape) < 0.05] = 0.0
    d[h // 5:h // 5 + 180, w // 6:w // 6 + 300] = 0.0
    tie = (slice(h // 2, h), slice(w // 2, w))
    d[tie] = np.where(d[tie] > 0, np.round(d[tie] * 8.0) / 8.0, 0.0)
    return d


@pytest.mark.parametrize("scale", [7, 8])
def test_set_scale_bitwise(scale):
    """StereoView::set_scale at blur radius 45 (scale 7) and 90 (scale 8):
    colour views through the three kernels; grey float images through the
    TMA-staged kernel at scale 7 and, its tile too large for shared memory,
    the three kernels at scale 8; byte images at a width whose rows are not
    16-byte aligned (three kernels) and at one whose rows are (TMA)."""
    sc = colour_scene(W, H, 2, 140 + scale)
    R = oref.RefScene(sc)
    try:
        R.set_scale(scale)
        with api.Context(0) as ctx:
            for v in range(3):
                blur, grad, hess = ctx.view_set_scale(R.image(v), scale)
                assert np.array_equal(blur, R.scaleimage(v)), v
                assert np.array_equal(grad, R.gradients(v)), v
                assert np.array_equal(hess, R.hessian(v)), v
    finally:
        R.close()
    for w in (1300, 1296):
        g = synth.make_scene(w, H, 1, seed_index=150 + scale)
        R = oref.RefScene(g)
        try:
            R.set_scale(scale)
            Mi, ti = R.Mt()
            with api.Context(0) as ctx:
                ctx.set_views_u8(scale, g.images[0], g.images[1:], Mi, ti, R.flen(0),
                                 R.inverse_flen(0))
                assert np.array_equal(ctx.debug_get_view(0)[0], R.gradients(0)), w
                gs, hs = ctx.debug_get_view(1)
                assert np.array_equal(gs, R.gradients(1)), w
                assert np.array_equal(hs, R.hessian(1)), w
                blur, grad, hess = ctx.view_set_scale(R.image(1), scale)
                assert np.array_equal(blur, R.scaleimage(1)), w
                assert np.array_equal(grad, R.gradients(1)), w
                assert np.array_equal(hess, R.hessian(1)), w
        finally:
            R.close()


@pytest.mark.parametrize("scale", [7, 8])
def test_surface_create_subdivide_fill(scale):
    """Surface::create from a depth map at scale 7 / 8 (node medians over
    windows of 16 K / 64 K depths), then subdivision down to scale 6 with
    fill_patches_from_depth after each step: node flags, patch flags and node
    values EQUAL to the reference's."""
    sc = synth.make_scene(W, H, 2, seed_index=160 + scale)
    init = _init_depth(sc, scale)
    R = oref.RefScene(sc)
    ctx = _ctx_with_sizes(R, 2)
    try:
        R.surface_create(scale, init)
        ctx.surface_create(scale, init)
        _assert_surface_equal(ctx, R, f"create {scale}")
        assert ctx.surface_state()[1].mean() > 0.3
        for s in range(scale - 1, 5, -1):
            R.surface_subdivide()
            ctx.surface_subdivide()
            _assert_surface_equal(ctx, R, f"subdivide to {s}")
            R.surface_fill_from_depth()
            ctx.surface_fill_from_depth()
            _assert_surface_equal(ctx, R, f"fill at {s}")
    finally:
        ctx.close()
        R.close()


@pytest.mark.parametrize("scale", [7, 8])
def test_construct_and_newton_loop(scale):
    """GaussNewtonStep::construct with 1024 / 4096 samples per patch
    (gradient, Hessian blocks and preconditioner in the reference's layout),
    then a whole Newton loop: same step count, CG iterations and active set,
    the same depth map to fp32 rounding."""
    P = Pair(W, H, 3, scale, seed_index=170 + scale)
    try:
        rng = np.random.default_rng(scale)
        full = P.node_valid.copy()
        part = (full & (rng.random(full.shape) < 0.5)).astype(np.uint8)
        for act, reg in ((full, 0.01), (part, 0.01), (full, 0.0)):
            P.R.gn_construct(act, None, reg, 0.0)
            P.ctx.gn_construct(act, None, reg, 0.0)
            assert_system_equal(P.ctx.debug_get_system(), P.R.get_system())
        sr = P.R.newton_loop(None, 0.01, 0.0)
        sg = P.ctx.newton_loop(None, 0.01, 0.0)
        for k in ("newton_steps", "cg_iterations", "n_active", "pixel_iterations"):
            assert sg[k] == sr[k], k
        assert sr["newton_steps"] > 1
        d, dr = P.ctx.get_depth(), P.R.surface_depth()
        assert np.array_equal(d > 0, dr > 0) and rel_err(d, dr) < 1e-6
    finally:
        P.close()


@pytest.mark.parametrize("scale", [7, 8])
@pytest.mark.parametrize("use_sgm", [True, False])
def test_visibility_and_cut(scale, use_sgm):
    """DepthOptimizer::create_subview_surfaces in both modes (the NCC filter
    walks a 128 / 256 pixel patch and its rim) and cut_boundaries: deleted
    patches, nodes and visibility lists EQUAL to the reference's."""
    n_sub = 4
    sc = colour_scene(W, H, n_sub, 180 + scale)
    init = sc.init_depth.astype(np.float32).copy()
    init[H // 3:H // 2 + 100, W // 3:W // 2 + 150] *= 0.8
    init[H // 2 + 60:H - 100, W // 10:W // 4] *= 1.15
    yy, xx = np.mgrid[0:H, 0:W]
    sgm = sc.init_depth.astype(np.float32).copy()
    sgm[(xx - 0.7 * W) ** 2 + (yy - 0.6 * H) ** 2 < (0.15 * H) ** 2] *= 0.6
    sgm[(xx + 2 * yy) % 17 == 0] = 0.0
    R = oref.RefScene(sc)
    try:
        R.set_scale(scale)
        R.surface_create(scale, init)
        if use_sgm:
            R.set_sgm_depth(sgm)
        info = R.surface_info()
        nodes, nv, pv = R.surface_get()
        Mi, ti = R.Mt()
        with api.Context(0) as ctx:
            ctx.set_views(R.gradients(0), [R.gradients(k + 1) for k in range(n_sub)],
                          [R.hessian(k + 1) for k in range(n_sub)], Mi, ti,
                          R.flen(0), R.inverse_flen(0))
            ctx.set_surface(info["scale"], info["npx"], info["npy"], info["start_x"],
                            info["start_y"], nodes, nv, pv, None, None)
            if not use_sgm:
                ctx.set_color_images(R.image(0), [R.image(k + 1) for k in range(n_sub)])
            left = R.create_subview_surfaces(use_sgm)
            removed = ctx.visibility(sgm if use_sgm else None)
            _, nv_r, pv_r = R.surface_get()
            off_r, ids_r = R.get_visibility()
            nv_g, pv_g, off_g, ids_g = ctx.surface_state()
            assert np.array_equal(pv_g, pv_r) and np.array_equal(nv_g, nv_r)
            assert int(pv.sum()) - removed == left == int(pv_g.sum())
            assert left > 0
            assert _lists(off_r, ids_r, pv_r) == _lists(off_g, ids_g, pv_g)
            K = R.inverse_calibration()
            for _ in range(6):
                d_r = R.cut_boundaries()
                d_g = ctx.cut_boundaries(K)
                _, nv_r, pv_r = R.surface_get()
                nv_g, pv_g, _, _ = ctx.surface_state()
                assert d_g == d_r
                assert np.array_equal(pv_g, pv_r) and np.array_equal(nv_g, nv_r)
                if d_r == 0:
                    break
    finally:
        R.close()


def _ladder(width, height, min_scale, seed, start_scale, cached=None):
    """The resident optimize() without SGM against RefScene.optimize_nosgm,
    under the bounds of test_resident_optimize_without_sgm. cached: the
    reference's (sparse depth, depth map) for this scene, if already known."""
    sc = colour_scene(width, height, 3, seed)
    R = oref.RefScene(sc)
    try:
        if cached is None:
            feats = _features_on_surface(sc, 2000, seed)
            sparse, d_cpu, _ = R.optimize_nosgm(feats, regularization=0.01,
                                                num_iterations=5, min_scale=min_scale)
        else:
            sparse, d_cpu = cached
        Mi, ti = R.Mt()
        imgs = [R.image(v) for v in range(4)]
        with api.Context(0) as ctx:
            d, _, _, st = api.optimize(ctx, imgs[0], imgs[1:], Mi, ti, R.flen(0),
                                       R.inverse_flen(0), R.inverse_calibration(), sparse,
                                       min_scale=min_scale, use_sgm=False)
    finally:
        R.close()
    assert st["final_scale"] == min_scale
    assert st["scales"] == start_scale - min_scale + 1
    assert np.array_equal(d_cpu > 0, d > 0)
    m = d_cpu > 0
    assert m.mean() > 0.15, m.mean()
    rel = np.abs(d[m] - d_cpu[m]) / d_cpu[m]
    print({"rel_median": float(np.median(rel)), "rel_max": float(rel.max())})
    assert float(np.median(rel)) < 1e-6
    assert rel.max() < 1e-3, rel.max()


def test_ladder_from_scale_7():
    """3200 x 2200 (7.04 MP) without SGM starts at scale 7."""
    _ladder(3200, 2200, 6, 190, 7)


def test_ladder_from_scale_8(ladder8_reference):
    """6400 x 4300 (27.5 MP) without SGM starts at scale 8; the reference's
    result comes from benchmarks/highres_cpu.py (cached)."""
    job = hc.LADDER8
    ref = ladder8_reference()
    _ladder(job["width"], job["height"], job["min_scale"], job["seed"], 8,
            cached=(ref["sparse"], ref["depth"]))


@pytest.mark.skipif(not os.path.exists(oref.INTEGRATION_LIB_PATH),
                    reason="oracle/_ref/integration not built")
def test_drop_in_optimize_from_scale_7():
    """The reference's unmodified optimize() through the drop-in build on the
    3200 x 2200 scene without SGM: the resident path takes the view from
    scale 7 and returns what the pure-CPU build returns."""
    sc = colour_scene(3200, 2200, 3, 192)
    feats = _features_on_surface(sc, 2000, 192)
    out = []
    for path in (None, oref.INTEGRATION_LIB_PATH):
        R = oref.RefScene(sc, lib_path=path)
        before = api.lib().smvsb_global_launch_count()
        try:
            _, d, _ = R.optimize_nosgm(feats, regularization=0.01, num_iterations=5,
                                       min_scale=6)
        finally:
            R.close()
        assert (api.lib().smvsb_global_launch_count() - before > 20) == (path is not None)
        out.append(d)
    d_cpu, d_gpu = out
    assert np.array_equal(d_cpu > 0, d_gpu > 0)
    m = d_cpu > 0
    assert m.mean() > 0.15, m.mean()
    rel = np.abs(d_gpu[m] - d_cpu[m]) / d_cpu[m]
    assert float(np.median(rel)) < 1e-6
    assert rel.max() < 1e-3, rel.max()


def test_scale_9_is_refused():
    """Scale 9 (above 108.8 MP without SGM) stays out of range, and the error
    names the limit."""
    sc = synth.make_scene(W, H, 1, seed_index=193)
    R = oref.RefScene(sc)
    try:
        with _ctx_with_sizes(R, 1) as ctx:
            for call in (lambda: ctx.surface_create(9, sc.init_depth),
                         lambda: ctx.set_surface(9, 2, 2, 0, 0, np.zeros(36),
                                                 np.ones(9, np.uint8),
                                                 np.ones(4, np.uint8), None, None)):
                with pytest.raises(api.SmvsbError) as e:
                    call()
                assert e.value.code == -1 and "0..8" in str(e.value)
    finally:
        R.close()
