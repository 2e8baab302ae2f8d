"""The image-side kernels at tiny, ragged and colour shapes, the rendered maps
at every scale, the lighting fit against an exact solve, SGM at its smallest
images and Gauss-Newton on degenerate patch grids.

Every comparison is bitwise, except the Gauss-Newton system (the tolerances
of test_gpu_parity.assert_system_equal) and the lighting fit, whose bounds are
derived in the docstrings of its tests.

  * set_scale (views.cu): the TMA-staged fused kernel (row pitch a multiple
    of 16 bytes: u8 widths % 16 == 0, float widths % 4 == 0) and the three
    kernels, for images shorter and narrower than one 64x32 tile and than the
    blur radius (12 at scale 5, 45 at 7, 90 at 8), 3 to 5 rows (the stencil's
    zero border), and one tile +- 1 pixel; against the numpy mirror
    smvs_b200.stereo_view, itself pinned here to the compiled reference at
    the same shapes. Images under 3x3 are refused.
  * the joint bilateral filter: colour guides and odd half-size depth maps
    against the compiled reference, every kernel size, channel count and
    guide range against the restatement oracle.port (pinned to the reference
    first), including guides whose values lie more than 3.77 apart, where the
    range weight's expf underflows to 0.
  * depth and normal maps (render_kernel) of surfaces created on both sides
    at scales 0-8, with holes, and of a single patch.
  * smvsb_fit_lighting and the reference's fit against an mpmath solve of the
    exactly summed normal equations.
  * SGM at 31..129 columns and 8..17 rows, single, reconstruct and banded.
  * gn_construct / cg_solve / update_nodes on grids one patch wide, one patch
    tall and of a single patch.
"""
import ctypes as C
import math

import numpy as np
import pytest

from smvs_b200 import api, stereo_view, synth
from oracle import port as oport
from oracle import ref as oref

from util_scene import Pair, colour_scene, rel_err

needs_ref = pytest.mark.skipif(not oref.available(), reason="oracle/_ref not built")
gpu = pytest.mark.gpu

SCALES = range(9)
ERR_INVALID = -1          # SMVSB_ERR_INVALID
ERR_STATE = -4            # SMVSB_ERR_STATE


def _noise_u8(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, size=shape, dtype=np.uint8)


# ---------------------------------------------------------------------------
# 1. set_scale at small and ragged shapes
# ---------------------------------------------------------------------------

U8_WIDTHS = (15, 16, 17, 32, 63, 64, 65, 128, 1024)      # TMA for w % 16 == 0
F32_WIDTHS = (3, 4, 5, 8, 15, 16, 17, 63, 64, 65, 1024)  # TMA for w % 4 == 0
HEIGHTS = (3, 4, 5, 31, 32, 33, 65)                      # 65: one tile + one row
RGB_WIDTHS = (3, 4, 17, 64, 65)
RGB_HEIGHTS = (3, 5, 33, 65)
REFUSED = ((16, 1), (16, 2), (1, 16), (2, 16), (2, 2))   # (w, h) under 3x3


@needs_ref
@pytest.mark.parametrize("w", (3, 15, 16, 17, 65))
def test_set_scale_mirror_matches_reference_at_small_shapes(w):
    """The numpy mirror the device tests compare with, against the compiled
    reference (StereoView::set_scale) at the small shapes those tests use,
    every scale: blurred image, gradients and Hessian bitwise."""
    for h in (3, 4, 5, 33, 65):
        sc = synth.make_scene(w, h, 1, seed_index=300 + w + h)
        R = oref.RefScene(sc)
        try:
            for scale in SCALES:
                R.set_scale(scale)
                for v in (0, 1):
                    b, g, hs = stereo_view.set_scale(sc.images[v], scale)
                    assert np.array_equal(b, R.scaleimage(v)), (w, h, scale, v)
                    assert np.array_equal(g, R.gradients(v)), (w, h, scale, v)
                    assert np.array_equal(hs, R.hessian(v)), (w, h, scale, v)
        finally:
            R.close()


@needs_ref
def test_set_scale_mirror_matches_reference_colour_small_shapes():
    for (w, h) in ((3, 3), (17, 5), (64, 33), (65, 65)):
        sc = colour_scene(w, h, 1, 310 + w)
        R = oref.RefScene(sc)
        try:
            for scale in SCALES:
                R.set_scale(scale)
                b, g, hs = stereo_view.set_scale(sc.images[1], scale)
                assert np.array_equal(b, R.scaleimage(1)), (w, h, scale)
                assert np.array_equal(g, R.gradients(1)), (w, h, scale)
                assert np.array_equal(hs, R.hessian(1)), (w, h, scale)
        finally:
            R.close()


@gpu
@pytest.mark.parametrize("scale", SCALES)
def test_set_views_u8_small_and_ragged(scale):
    """smvsb_set_views_u8 at every (width, height) of U8_WIDTHS x HEIGHTS,
    each image once as a neighbour (gradients and Hessian) and the first of
    each call also as the main view (gradients): bitwise the mirror."""
    shapes = [(w, h) for w in U8_WIDTHS for h in HEIGHTS]
    imgs = [_noise_u8((h, w), 1000 * scale + i) for i, (w, h) in enumerate(shapes)]
    with api.Context(0) as ctx:
        for lo in range(0, len(imgs), 31):
            chunk = imgs[lo:lo + 31]
            n = len(chunk)
            Mi = np.tile(np.eye(3).ravel(), (n, 1))
            ti = np.tile([0.1, 0.0, 0.0], (n, 1))
            ctx.set_views_u8(scale, chunk[0], chunk, Mi, ti, 100.0, 0.01)
            g, _ = ctx.debug_get_view(0)
            assert np.array_equal(g, stereo_view.set_scale(chunk[0], scale)[1])
            for k, img in enumerate(chunk):
                _, rg, rh = stereo_view.set_scale(img, scale)
                g, hs = ctx.debug_get_view(k + 1)
                assert np.array_equal(g, rg), (img.shape, scale)
                assert np.array_equal(hs, rh), (img.shape, scale)


@gpu
@pytest.mark.parametrize("scale", SCALES)
def test_view_set_scale_f32_and_rgb_small_and_ragged(scale):
    """smvsb_view_set_scale_c with one float channel (TMA-staged for widths
    % 4 == 0) and with three (always the three kernels): scaleimage,
    gradients and Hessian bitwise the mirror."""
    with api.Context(0) as ctx:
        for i, (w, h) in enumerate((w, h) for w in F32_WIDTHS for h in HEIGHTS):
            img = _noise_u8((h, w), 2000 * scale + i)
            blur, grad, hess = ctx.view_set_scale(stereo_view.byte_to_float(img), scale)
            rb, rg, rh = stereo_view.set_scale(img, scale)
            assert np.array_equal(blur, rb), (w, h, scale)
            assert np.array_equal(grad, rg), (w, h, scale)
            assert np.array_equal(hess, rh), (w, h, scale)
        for i, (w, h) in enumerate((w, h) for w in RGB_WIDTHS for h in RGB_HEIGHTS):
            img = _noise_u8((h, w, 3), 3000 * scale + i)
            blur, grad, hess = ctx.view_set_scale(stereo_view.byte_to_float(img), scale)
            rb, rg, rh = stereo_view.set_scale(img, scale)
            assert np.array_equal(blur, rb), (w, h, scale)
            assert np.array_equal(grad, rg), (w, h, scale)
            assert np.array_equal(hess, rh), (w, h, scale)


@gpu
@pytest.mark.parametrize("w,h", REFUSED)
def test_set_scale_refuses_images_under_3x3(w, h):
    """Under 3x3 there is no interior for the stencil: both entry points fail
    with SMVSB_ERR_INVALID and a message, write nothing to the caller's
    buffers, and leave the context without views."""
    L = api.lib()
    img = _noise_u8((h, w), 7)
    ok = _noise_u8((8, 16), 8)
    Mi, ti = np.eye(3).ravel()[None], np.zeros((1, 3))
    with api.Context(0) as ctx:
        for main, sub in ((img, ok), (ok, img)):
            with pytest.raises(api.SmvsbError) as e:
                ctx.set_views_u8(2, main, [sub], Mi, ti, 100.0, 0.01)
            assert e.value.code == ERR_INVALID and str(e.value).split(":", 1)[1].strip()
            with pytest.raises(api.SmvsbError) as e:
                ctx.debug_get_view(0)
            assert e.value.code == ERR_STATE
        for ch in (1, 3):
            f = np.ascontiguousarray(np.full((h, w, ch), 0.5, np.float32))
            outs = [np.full(h * w * k, np.nan, np.float32) for k in (ch, 2, 3)]
            rc = L.smvsb_view_set_scale_c(ctx._h, w, h, ch, f.ctypes.data_as(C.c_void_p), 2,
                                          *[o.ctypes.data_as(C.c_void_p) for o in outs])
            assert rc == ERR_INVALID
            assert L.smvsb_last_error(ctx._h)
            assert all(np.isnan(o).all() for o in outs)


# ---------------------------------------------------------------------------
# 2. the joint bilateral filter
# ---------------------------------------------------------------------------

def _with_holes(d, seed):
    rng = np.random.default_rng(seed)
    d = np.array(d, dtype=np.float32, copy=True)
    h, w = d.shape
    d[rng.random(d.shape) < 0.05] = 0.0
    d[h // 4:h // 4 + max(1, h // 5), w // 3:w // 3 + max(1, w // 4)] = 0.0
    return d


@gpu
@needs_ref
def test_bilateral_colour_guide_matches_reference():
    """DepthOptimizer::depthmap_bilateral_filter with the three-channel image
    of a colour view as guide (what every MVE scene has): full-size depth and
    the two half-size depth maps of an odd image, (w + 1) // 2 x (h + 1) // 2
    and w // 2 x h // 2, with holes. The restatement oracle.port agrees with
    the reference on the same inputs, which the parameter sweep relies on."""
    sc = colour_scene(333, 207, 1, 41)
    R = oref.RefScene(sc)
    try:
        guide = R.image(0)
        assert guide.shape == (207, 333, 3)
        full = _with_holes(sc.init_depth, 1)
        maps = (full, _with_holes(sc.init_depth[::2, ::2], 2),
                _with_holes(sc.init_depth[1::2, 1::2], 3))
        assert [m.shape for m in maps] == [(207, 333), (104, 167), (103, 166)]
        with api.Context(0) as ctx:
            for dm in maps:
                ref = R.bilateral_filter(dm)
                assert np.array_equal(ctx.bilateral_filter(guide, dm), ref), dm.shape
                assert np.array_equal(oport.bilateral_filter(guide, dm), ref), dm.shape
                assert (ref > 0).mean() > 0.8
    finally:
        R.close()


def _guides(seed):
    """Guides of 1..4 channels: a 61x47 crop of a colour view (extra channels
    from its luminance), and a 5x3 one, smaller than every window but k = 0, 1."""
    sc = colour_scene(61, 47, 1, seed)
    rgb = stereo_view.byte_to_float(sc.images[0])
    lum = stereo_view.desaturate_luminance(rgb)[..., None]
    four = np.concatenate([rgb, lum], axis=2)
    out = []
    for ch in (1, 2, 3, 4):
        g = four[:, :, :ch] if ch > 1 else four[:, :, 3]
        out += [np.ascontiguousarray(g), np.ascontiguousarray(g[20:23, 30:35])]
    return out, sc.init_depth


@gpu
@needs_ref
def test_bilateral_parameter_sweep_matches_restatement():
    """kernel_size 0..8, sigma 0.5 / 5 / 20, 1..4 guide channels, guides
    narrower and shorter than the window, depth maps smaller and larger than
    the guide: bitwise oracle.port.bilateral_filter (libm's expf), which is
    pinned to the reference at the default parameters first."""
    sc = synth.make_scene(61, 47, 1, seed_index=42)
    R = oref.RefScene(sc)
    try:
        d = _with_holes(sc.init_depth, 4)
        assert np.array_equal(oport.bilateral_filter(R.image(0), d), R.bilateral_filter(d))
    finally:
        R.close()
    guides, depth = _guides(43)
    with api.Context(0) as ctx:
        for g in guides:
            h, w = g.shape[:2]
            maps = (_with_holes(depth[:h, :w], 5),                    # same size
                    _with_holes(depth[: (h + 1) // 2, : (w + 1) // 2], 6),
                    _with_holes(np.tile(depth, (2, 2))[: 2 * h + 1, : 3 * w], 7))
            for dm in maps:
                for ks in range(9):
                    for sigma in (0.5, 5.0, 20.0):
                        out = ctx.bilateral_filter(g, dm, sigma, ks)
                        ref = oport.bilateral_filter(g, dm, sigma, ks)
                        assert np.array_equal(out, ref), (g.shape, dm.shape, ks, sigma)


@gpu
@pytest.mark.parametrize("lo,hi", [(-1.0, 2.0), (0.0, 255.0)])
def test_bilateral_wide_range_guide(lo, hi):
    """Float guides through the C ABI need not lie in [0, 1]. Two guide values
    more than 3.77 apart give a range argument below glibc's underflow bound
    (-diff^2 / 0.02 < -103.97), where expf is 0: the weight is 0, not inf or
    NaN, and the output is bitwise the restatement's (libm's expf)."""
    rng = np.random.default_rng(int(hi))
    sc = synth.make_scene(61, 47, 1, seed_index=44)
    d = _with_holes(sc.init_depth, 8)
    with api.Context(0) as ctx:
        for ch in (1, 3):
            g = (lo + (hi - lo) * rng.random((47, 61, ch))).astype(np.float32)
            g[10:20, 10:20] = np.float32(lo)         # flat region: weights survive
            g = np.ascontiguousarray(g if ch > 1 else g[:, :, 0])
            for ks in (1, 5, 8):
                out = ctx.bilateral_filter(g, d, 5.0, ks)
                ref = oport.bilateral_filter(g, d, 5.0, ks)
                assert np.isfinite(out).all()
                assert np.array_equal(out, ref), (ch, ks)


# ---------------------------------------------------------------------------
# 3. depth and normal maps at every scale
# ---------------------------------------------------------------------------

# (scale, width, height): odd sizes, grids that end short of the right and
# bottom edges; (5, 71, 67) is a single patch
MAP_CASES = [(0, 97, 71), (1, 97, 71), (2, 133, 101), (3, 203, 157), (4, 333, 207),
             (5, 333, 207), (6, 467, 333), (7, 645, 519), (8, 1031, 777), (5, 71, 67),
             (8, 601, 533)]


@gpu
@needs_ref
@pytest.mark.parametrize("scale,w,h", MAP_CASES)
def test_depth_and_normal_maps_every_scale(scale, w, h):
    """Surface::create from a depth map with holes (scale 0: create at 1 and
    subdivide, the only way the reference makes a scale-0 surface) on both
    sides, then Surface::get_depth_map and get_normal_map(inv_flen): both
    bitwise. The focal length 0.93 * max(w, h) has no exact float inverse,
    and the device is given inv_flen as a double that narrows to the
    reference's float: get_normal_map takes a float."""
    sc = synth.make_scene(w, h, 1, seed_index=50 + scale)
    sc.flen = np.float32([0.93, 1.0])
    init = _with_holes(sc.init_depth, scale)
    R = oref.RefScene(sc)
    try:
        R.set_scale(2)
        inv_flen = R.inverse_flen(0)
        assert inv_flen != 1.0 / R.flen(0)
        inv_wide = inv_flen * (1.0 + 2.0 ** -40)
        assert np.float32(inv_wide) == np.float32(inv_flen) and inv_wide != inv_flen
        with api.Context(0) as ctx:
            ctx.set_views_u8(2, sc.images[0], sc.images[1:], *R.Mt(), R.flen(0), inv_wide)
            R.surface_create(max(scale, 1), init)
            ctx.surface_create(max(scale, 1), init)
            if scale == 0:
                R.surface_subdivide()
                ctx.surface_subdivide()
            info = R.surface_info()
            assert ctx.surface_info() == info
            ps, npx, npy = info["patchsize"], info["npx"], info["npy"]
            assert info["start_x"] + npx * ps < w and info["start_y"] + npy * ps < h
            if (w, h) in ((71, 67), (601, 533)):
                assert npx == npy == 1
            nodes, nv, pv = R.surface_get()
            gn = ctx.get_nodes()
            gnv, gpv, _, _ = ctx.surface_state()
            assert np.array_equal(gnv, nv) and np.array_equal(gpv, pv)
            assert np.array_equal(gn[nv != 0], nodes[nv != 0])
            assert pv.any()
            depth, rdepth = ctx.get_depth(), R.surface_depth()
            assert np.array_equal(depth, rdepth)
            normals, rnormals = ctx.get_normals(), R.surface_normals()
            bad = np.argwhere(normals != rnormals)
            assert bad.size == 0, (len(bad), bad[:5])
    finally:
        R.close()


# ---------------------------------------------------------------------------
# 4. the lighting fit against an exact solve
# ---------------------------------------------------------------------------

U64 = 2.0 ** -53          # unit roundoff of double
U32 = 2.0 ** -24          # unit roundoff of float
SH_ROUNDINGS = 8          # roundings in the deepest SH term and its product


def _mpmath():
    try:
        import mpmath
    except ImportError:
        pytest.skip("mpmath (a dependency of sympy) is not installed")
    return mpmath


def _sh_of(normals):
    """sh::evaluate_4_band of the float normals widened to double."""
    return synth.sh_basis(np.asarray(normals, dtype=np.float64))


def _kept(normals, image):
    """LightOptimizer::fit_lighting_to_image's pixel rule: |norm(n) - 1| <=
    1e-6 with norm as math::Vector sums it (in double, from 0, in order) and
    image >= 0.05f."""
    n = np.asarray(normals, dtype=np.float64).reshape(-1, 3)
    length = np.sqrt(n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1] + n[:, 2] * n[:, 2])
    return (np.abs(length - 1.0) <= 1e-6) & (np.asarray(image).reshape(-1) >= np.float32(0.05))


def _split(a):
    """Veltkamp split: a = hi + lo, each with at most 26 significant bits, so
    that a product of two halves is exact in double."""
    c = a * 134217729.0                    # 2^27 + 1
    hi = c - (c - a)
    return hi, a - hi


def _exact_sum_of_products(a, b):
    """sum(a * b) correctly rounded: the four exact half products, fsum."""
    ah, al = _split(a)
    bh, bl = _split(b)
    return math.fsum(np.concatenate([ah * bh, ah * bl, al * bh, al * bl]))


def _normal_equations(normals, image):
    """A = sum sh sh^T and b = sum sh * I over the kept pixels, each entry
    the correctly rounded exact sum."""
    keep = _kept(normals, image)
    sh = _sh_of(normals.reshape(-1, 3)[keep])
    img = np.asarray(image, dtype=np.float32).reshape(-1)[keep].astype(np.float64)
    A = np.empty((16, 16))
    for i in range(16):
        for j in range(i, 16):
            A[i, j] = A[j, i] = _exact_sum_of_products(sh[:, i], sh[:, j])
    b = np.array([_exact_sum_of_products(sh[:, i], img) for i in range(16)])
    return A, b, keep, sh, img


def _exact_solve(A, b):
    """math::matrix_pseudo_inverse(A) * b in 40-digit arithmetic, singular
    values under 1e-12 dropped like MATH_EPSILON_EQ(s, 0, 1e-12) does.
    Returns (x, condition number, smallest singular value)."""
    mp = _mpmath()
    with mp.workdps(40):
        Am = mp.matrix(A.tolist())
        U, S, V = mp.svd_r(Am)
        inv = [mp.mpf(0) if abs(s) <= mp.mpf("1e-12") else 1 / s for s in S]
        Utb = U.T * mp.matrix(b.tolist())
        y = mp.matrix([Utb[i] * inv[i] for i in range(16)])
        x = V.T * y
        smax, smin = max(S), min(S)
        return (np.array([float(v) for v in x]), float(smax / smin), float(smin))


def _rounding_bound(kappa, depth):
    """Relative 2-norm error bound of a fit whose normal-equation sums have
    `depth` additions on the longest path to each entry (rounding error
    analysis of recursive summation, Higham, Accuracy and Stability, 4.2):

      each entry of A and b is a sum of terms sh_i sh_j (resp. sh_i I) that
      each carry SH_ROUNDINGS roundings, so |dA| <= gamma(depth + 8) * sum
      |sh||sh|^T elementwise; that sum's 2-norm is at most sum ||sh||^2 =
      trace(A) <= 16 ||A||, hence ||dA|| / ||A|| <= 16 gamma(depth + 8), and
      likewise ||db|| / ||b|| (I >= 0.05 and the constant band sh_0 = 1 keep
      ||b|| from cancelling: the kept terms of b_0 are all positive).
      The pseudo-inverse of the one-sided Jacobi SVD (both the host's
      pseudo_inverse_16 and the reference's) is backward stable with
      ||dA|| <= n^2 u ||A|| = 256 u ||A||, and the product A^+ b adds n u = 16 u
      relative in the worst case times kappa.

    Perturbation theory for A x = b then gives
      ||x^ - x|| / ||x|| <= kappa (eps_A + eps_b + 256 u + 16 u) / (1 - kappa eps_A)
    with eps = 16 gamma(depth + 8), gamma(k) = k u / (1 - k u); c is the
    bracket over u."""
    k = depth + SH_ROUNDINGS
    gamma = k * U64 / (1 - k * U64)
    eps = 16 * gamma
    assert kappa * eps < 0.5, "system too ill-conditioned for the bound"
    return kappa * (2 * eps + 272 * U64) / (1 - kappa * eps)


def _device_sum_depth(npix):
    """Additions on the longest path of light_partials_kernel + the host sum:
    a thread's strided pixels, 5 shuffle levels, 8 warps, then the grid's
    block partials in order (grid = min(4 SMs, ceil(npix / 256)))."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    grid = max(1, min(sms * 4, -(-npix // 256)))
    return -(-npix // (grid * 256)) + 5 + 8 + grid


def _bowl_nodes(w, h, scale, a=3e-3, depth0=3.0):
    """Node values (f, dx, dy, dxy in patch units) of w = depth0 + a r^2 about
    the image centre: a paraboloid cap the bicubic patches reproduce exactly,
    whose normals tilt up to ~70 degrees from the axis in every direction."""
    ps, npx, npy, sx, sy = synth.surface_grid(w, h, scale)
    iy, ix = np.mgrid[0:npy + 1, 0:npx + 1]
    u = (sx + ix * ps).astype(np.float64) - 0.5 * w
    v = (sy + iy * ps).astype(np.float64) - 0.5 * h
    f = depth0 + a * (u * u + v * v)
    nodes = np.stack([f, 2 * a * u * ps, 2 * a * v * ps, np.zeros_like(f)], axis=-1)
    return (ps, npx, npy, sx, sy), np.ascontiguousarray(nodes.reshape(-1, 4))


LIGHT_STAR = np.array([0.8, 0.1, 0.3, -0.1, 0.05, 0.02, 0.05, -0.03, 0.02, 0.01,
                       -0.01, 0.01, 0.005, -0.005, 0.004, 0.003])


@needs_ref
def test_sh_basis_is_the_references():
    """synth.sh_basis (vectorised) against sh::evaluate_4_band of the
    reference, bitwise, on normals of every direction."""
    rng = np.random.default_rng(60)
    n = rng.normal(size=(400, 3))
    n = (n / np.linalg.norm(n, axis=1, keepdims=True)).astype(np.float32).astype(np.float64)
    got = _sh_of(n)
    for k in range(len(n)):
        assert np.array_equal(got[k], oref.Units.sh_4band(n[k])[0]), k


@gpu
@needs_ref
def test_fit_lighting_known_answer():
    """A surface set directly (a paraboloid cap) and a shading image
    I = float(SH(n) . L*) from the device's own normal map: the fit must be
    the exact solution of the exact normal equations within the rounding
    bound of _rounding_bound, and that solution must be L* within what
    rounding I to float allows: with S the kept rows sh_p and delta_p =
    I_p - sh_p . L*, x - L* = S^+ delta, so ||x - L*|| <= ||delta|| /
    sigma_min(S) = ||delta|| / sqrt(lambda_min(A)), and |delta_p| <= u_f |I_p|
    + gamma(16) sum_i |sh_pi L*_i| (the float rounding and the double dot
    product that preceded it)."""
    w, h, scale = 161, 121, 3
    sc = synth.make_scene(w, h, 1, seed_index=61)
    (ps, npx, npy, sx, sy), nodes = _bowl_nodes(w, h, scale)
    nn, npatch = (npx + 1) * (npy + 1), npx * npy
    R = oref.RefScene(sc)
    try:
        R.set_scale(2)
        grads = [R.gradients(0), R.gradients(1)]
        hess1 = R.hessian(1)
        Mi, ti = R.Mt()
        flen, inv_flen = R.flen(0), R.inverse_flen(0)
    finally:
        R.close()
    with api.Context(0) as ctx:
        def push(shading):
            ctx.set_views(grads[0], [grads[1]], [hess1], Mi, ti, flen, inv_flen, shading,
                          np.zeros((h, w, 2), np.float32))
            ctx.set_surface(scale, npx, npy, sx, sy, nodes, np.ones(nn, np.uint8),
                            np.ones(npatch, np.uint8), None, None)
        push(np.ones((h, w), np.float32))
        normals = ctx.get_normals()
        mask = np.abs(np.linalg.norm(normals.astype(np.float64), axis=2) - 1.0) <= 1e-6
        assert mask.mean() > 0.7
        assert normals[mask][:, 2].min() < 0.4          # normals spread widely
        shading = np.zeros((h, w), np.float32)
        shading[mask] = (_sh_of(normals[mask]) @ LIGHT_STAR).astype(np.float32)
        push(shading)
        assert np.array_equal(ctx.get_normals(), normals)
        fit = ctx.fit_lighting()
    A, b, keep, sh, img = _normal_equations(normals, shading)
    x, kappa, smin = _exact_solve(A, b)
    bound = _rounding_bound(kappa, _device_sum_depth(w * h))
    assert np.linalg.norm(fit - x) <= bound * np.linalg.norm(x), (fit - x, kappa, bound)
    gamma16 = 16 * U64 / (1 - 16 * U64)
    delta = U32 * np.abs(img) + gamma16 * (np.abs(sh) @ np.abs(LIGHT_STAR))
    star_bound = np.linalg.norm(delta) / math.sqrt(smin)
    assert np.linalg.norm(x - LIGHT_STAR) <= star_bound, (x - LIGHT_STAR, star_bound)
    assert np.linalg.norm(fit - LIGHT_STAR) <= star_bound + bound * np.linalg.norm(x)


@gpu
@needs_ref
def test_fit_lighting_scene_against_exact_solve():
    """The shading scene the parity tests fit (kappa ~ 1e8): the device's fit
    and the reference's, each against the exact solve within its own
    rounding bound -- the reference sums all pixels one after the other
    (depth = number of kept pixels), the device in a tree."""
    P = Pair(640, 480, 1, 2, shading=True)
    try:
        normals = P.R.surface_normals()
        assert np.array_equal(P.ctx.get_normals(), normals)
        image, _ = P.R.shading()
        fit, ref = P.ctx.fit_lighting(), P.R.fit_lighting()
    finally:
        P.close()
    A, b, keep, _, _ = _normal_equations(normals, image)
    x, kappa, _ = _exact_solve(A, b)
    assert kappa > 1e6
    dev_bound = _rounding_bound(kappa, _device_sum_depth(640 * 480))
    ref_bound = _rounding_bound(kappa, int(keep.sum()))
    nx = np.linalg.norm(x)
    assert np.linalg.norm(fit - x) <= dev_bound * nx, (np.linalg.norm(fit - x) / nx, dev_bound)
    assert np.linalg.norm(ref - x) <= ref_bound * nx, (np.linalg.norm(ref - x) / nx, ref_bound)


# ---------------------------------------------------------------------------
# 5. SGM at the smallest shapes
# ---------------------------------------------------------------------------

SGM_WIDTHS = (31, 32, 33, 63, 65, 127, 129)
SGM_HEIGHTS = range(8, 18)        # the census needs w > 9 and h > 7


@gpu
@needs_ref
@pytest.mark.parametrize("D", [32, 256])
@pytest.mark.parametrize("w", SGM_WIDTHS)
def test_sgm_smallest_shapes(w, D):
    """SGMStereo::run_sgm (cost and aggregated volumes, depth), reconstruct
    (both directions and the consistency check) and a run under a budget
    that allows bands of 16 rows only (two bands at 17 rows): bit-exact at
    widths around the 32-lane groups of the path kernels and heights from
    the census minimum to 17."""
    from test_gpu_sgm_budget import budget_for, expected_bands, volume_bytes
    for h in SGM_HEIGHTS:
        sc = synth.make_scene(w, h, 1, seed_index=70 + h)
        dmin, dmax = float(sc.true_depth.min() * 0.7), float(sc.true_depth.max() * 1.3)
        R = oref.RefScene(sc)
        try:
            r = R.sgm_run(0, 1, 0, D, dmin, dmax, volumes=True)
            rec = R.sgm_reconstruct(0, 1, 0, D, dmin, dmax)
            M, t = R.reprojection(0, 1, w, h, w, h)
            Mb, tb = R.reprojection(1, 0, w, h, w, h)
        finally:
            R.close()
        g = api.sgm(sc.images[0], sc.images[1], M, t, dmin, dmax, D, volumes=True)
        assert np.array_equal(g["cost"], r["cost"]), (w, h, D)
        assert np.array_equal(g["sgm"], r["sgm"]), (w, h, D)
        assert np.array_equal(g["depth"], r["depth"]), (w, h, D)
        gr = api.sgm_reconstruct(sc.images[0], sc.images[1], M, t, Mb, tb, (dmin, dmax),
                                 (dmin, dmax), D)
        assert np.array_equal(gr["depth"], rec), (w, h, D)
        budget = budget_for(w, h, D, 16, False)
        gb, st = api.sgm(sc.images[0], sc.images[1], M, t, dmin, dmax, D,
                         device_bytes=budget, return_stats=True)
        assert np.array_equal(gb["depth"], r["depth"]), (w, h, D, st)
        if h > 16:
            rows, _ = expected_bands(w, h, D, volume_bytes(w, h, D, 16, False))
            assert rows == 16 and st["banded"] == 1 and st["bands"] == 2, st


# ---------------------------------------------------------------------------
# 6. degenerate patch grids
# ---------------------------------------------------------------------------

# (scale, w, h): one patch wide, one patch tall, a single patch. A scale-0
# surface only arises by subdividing a scale-1 one, whose narrowest grid (6
# pixels) becomes four patches across at scale 0: the narrowest there is.
GRID_CASES = [(s, w, h) for s, (a, b) in ((0, (6, 41)), (2, (13, 61)), (4, (41, 161)),
                                          (7, (301, 701)))
              for (w, h) in ((a, b), (b, a), (a, a))]


def _every_patch_sees_every_neighbour(P):
    """The surface as created, before visibility (which deletes the edge
    patches of images this small), each patch with every neighbour in its
    visibility list."""
    R, n = P.R, P.scene.n_sub
    R.surface_create(max(P.scale, 1), P.scene.init_depth)
    if P.scale == 0:
        R.surface_subdivide()
    P.info = R.surface_info()
    P.nodes, P.node_valid, P.patch_valid = R.surface_get()
    counts = P.patch_valid.astype(np.uint32) * n
    P.vis_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint32)
    P.vis_ids = np.tile(np.arange(n, dtype=np.uint8), int(P.patch_valid.sum()))
    R.set_visibility(P.vis_off, P.vis_ids)
    P.push_surface()


@gpu
@needs_ref
@pytest.mark.parametrize("scale,w,h", GRID_CASES)
def test_degenerate_patch_grids(scale, w, h):
    """gn_construct + cg_solve + update_nodes on grids whose every patch lies
    on the grid's edge: the preconditioner's 3x3 stencil rows and the PCG
    row lists with missing neighbours. Systems within the parity tolerances,
    equal iteration counts and active sets."""
    from test_gpu_parity import assert_system_equal
    P = Pair(w, h, 2, scale, seed_index=80 + scale)
    try:
        _every_patch_sees_every_neighbour(P)
        i = P.info
        base = 4 if scale == 0 else 1
        assert min(i["npx"], i["npy"]) == base
        if w == h:
            assert i["npx"] == i["npy"] == base
        assert P.patch_valid.any() and (scale == 0 or P.patch_valid.all())
        nv = P.node_valid
        P.R.gn_construct(nv, None, 0.01, 0.0)
        P.ctx.gn_construct(nv, None, 0.01, 0.0)
        assert_system_equal(P.ctx.debug_get_system(), P.R.get_system())
        xr, itr, infr = P.R.cg_solve()
        itg, infg = P.ctx.cg_solve()
        assert (itg, infg) == (itr, infr)
        if itr > 0:
            assert rel_err(P.ctx.get_delta(), xr) < 1e-8
        ar, nr, _ = P.R.update_nodes(xr, nv)
        ag, ng, _ = P.ctx.update_nodes()
        assert ng == nr and np.array_equal(ag, ar)
    finally:
        P.close()
