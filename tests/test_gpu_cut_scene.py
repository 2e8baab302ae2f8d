"""smvsb_cut_depth_maps_multi: the cross-view cut of scenes larger than one
device -- target groups, source views streamed in chunks, 16x16 tiles that
skip source views they cannot project into, several workers -- against the
reference's own MeshGenerator::cut_depth_maps (oracle/_ref). The cut maps
must be EQUAL for every device list and memory cap."""
import ctypes as C
import os

import numpy as np
import pytest

from smvs_b200 import api
from oracle import ref as oref

from test_gpu_cutmaps import make_views

needs_oracle = pytest.mark.skipif(not oref.available(), reason="oracle/_ref not built")

W, H = 320, 240


def facade(x, y):
    return 5.0 + 0.2 * np.sin(0.7 * x) * np.cos(1.3 * y)


def facade_grad(x, y):
    return 0.2 * 0.7 * np.cos(0.7 * x) * np.cos(1.3 * y), -0.2 * 1.3 * np.sin(0.7 * x) * np.sin(1.3 * y)


def rot_y(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])


def render(R, c, flen, w, h, wall_z=None, rng=None, iters=20):
    """Depth (MVE convention) and world normals facing the camera of the
    surface a pinhole camera (world -> camera R, centre c) sees: the facade
    z = facade(x, y), or with wall_z the plane z = wall_z. Rays that miss
    (or hit behind the camera) get depth 0."""
    ys, xs = np.mgrid[0:h, 0:w]
    ax = flen * max(w, h)
    dirs_cam = np.stack([(xs + 0.5 - 0.5 * w) / ax, (ys + 0.5 - 0.5 * h) / ax,
                         np.ones_like(xs, dtype=np.float64)], axis=-1)
    dirs_cam /= np.linalg.norm(dirs_cam, axis=-1, keepdims=True)
    dirs = dirs_cam @ R
    with np.errstate(divide="ignore", invalid="ignore"):
        if wall_z is not None:
            tt = (wall_z - c[2]) / dirs[..., 2]
            nrm = np.zeros(dirs.shape)
            nrm[..., 2] = -np.sign(wall_z - c[2])
        else:
            tt = np.full((h, w), 5.0)
            for _ in range(iters):
                px, py = c[0] + tt * dirs[..., 0], c[1] + tt * dirs[..., 1]
                tt = (facade(px, py) - c[2]) / dirs[..., 2]
            px, py = c[0] + tt * dirs[..., 0], c[1] + tt * dirs[..., 1]
            gx, gy = facade_grad(px, py)
            nrm = -np.stack([-gx, -gy, np.ones_like(gx)], axis=-1)
            nrm /= np.linalg.norm(nrm, axis=-1, keepdims=True)
    bad = ~np.isfinite(tt) | (tt <= 0) | (tt > 40)
    d = np.where(bad, 0.0, tt).astype(np.float32)
    if rng is not None:
        d[rng.random(d.shape) < 0.01] = 0.0
        y0, x0 = int(rng.integers(0, h - 40)), int(rng.integers(0, w - 60))
        d[y0:y0 + 40, x0:x0 + 60] *= np.float32(0.93)
    return d, nrm.astype(np.float32)


def strip_scene(seed=5, n_facade=12, w=W, h=H, flen=2.0, spacing=1.0, iters=20):
    """Cameras along a facade (each overlapping a few neighbours, image borders
    cutting through the neighbours' tiles), two cameras facing away from it
    towards a wall behind them, and one oblique camera whose plane z_cam = 0
    passes through facade points the others see. Returns (flen, rot, trans,
    depths, normals, kinds)."""
    rng = np.random.default_rng(seed)
    cams = []
    for k in range(n_facade):
        cams.append(("facade", rot_y(rng.uniform(-0.03, 0.03)),
                     np.array([spacing * k, rng.uniform(-0.1, 0.1), rng.uniform(-0.1, 0.1)])))
    for k in (3, 7):
        cams.append(("away", rot_y(np.pi + rng.uniform(-0.03, 0.03)),
                     np.array([spacing * k + 0.3, 0.0, 0.5])))
    cams.append(("oblique", rot_y(-1.0), np.array([spacing * 4.0, 0.0, 3.0])))
    return render_views(cams, seed, flen, w, h, iters)


def ring_scene(n, w, h, seed, flen=1.1, iters=20):
    """n cameras on a circle of radius 0.6 in the plane z = 0, all looking at
    the facade: every view sees every other."""
    rng = np.random.default_rng(seed)
    cams = [("facade", rot_y(rng.uniform(-0.05, 0.05)),
             np.array([0.6 * np.cos(2 * np.pi * k / n), 0.6 * np.sin(2 * np.pi * k / n), 0.0]))
            for k in range(n)]
    return render_views(cams, seed, flen, w, h, iters)


def render_views(cams, seed, flen, w, h, iters):
    """Renders (kind, R, c) cameras on a thread pool, view k's disturbances
    seeded with (seed, k). Returns (flen, rot, trans, depths, normals, kinds)."""
    import concurrent.futures

    def one(k):
        kind, R, c = cams[k]
        R = R.astype(np.float32).astype(np.float64)
        t = (-R @ c).astype(np.float32).astype(np.float64)
        c = -R.T @ t
        d, nrm = render(R, c, flen, w, h, wall_z=-4.0 if kind == "away" else None,
                        rng=np.random.default_rng((seed, k)), iters=iters)
        return R.reshape(9), t, d, nrm

    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        res = list(ex.map(one, range(len(cams))))
    return (np.full(len(cams), flen, np.float32), np.array([r[0] for r in res], np.float32),
            np.array([r[1] for r in res], np.float32), [r[2] for r in res],
            [r[3] for r in res], [c[0] for c in cams])


def world_points(depth, inv, ctw):
    h, w = depth.shape
    ys, xs = np.mgrid[0:h, 0:w]
    px = np.stack([xs + 0.5, ys + 0.5, np.ones_like(xs, dtype=np.float64)], -1)
    ray = px @ inv.reshape(3, 3).astype(np.float64).T
    ray /= np.linalg.norm(ray, axis=-1, keepdims=True)
    M = ctw.reshape(4, 4).astype(np.float64)
    p = (ray * depth[..., None]) @ M[:3, :3].T + M[:3, 3]
    return p[depth != 0]


def projections(p, KR, t):
    return p @ KR.reshape(3, 3).astype(np.float64).T - t.astype(np.float64)


@pytest.fixture(scope="module")
def strip():
    flen, rot, trans, depths, normals, kinds = strip_scene()
    outs, inv, ctw, KR, t = oref.cut_depth_maps(flen, rot, trans, depths, normals)
    return dict(depths=depths, normals=normals, kinds=kinds, ref=outs, mats=(inv, ctw, KR, t))


def _equal(got, ref):
    assert len(got) == len(ref)
    for g, o in zip(got, ref):
        assert np.array_equal(g, o)


@needs_oracle
def test_strip_scene_populates_every_category(strip):
    """CPU: the scene has what the culling must get right, and the
    reference's cut keeps part of it."""
    inv, ctw, KR, t = strip["mats"]
    kinds, depths = strip["kinds"], strip["depths"]
    n = len(depths)
    pts = [world_points(d, inv[i], ctw[i]) for i, d in enumerate(depths)]
    near_edge = out_of_view = total = 0
    behind_away = straddle = 0
    for i in range(n):
        for j in range(n):
            if i == j:
                continue
            pr = projections(pts[i], KR[j], t[j])
            total += len(pr)
            z = pr[:, 2]
            with np.errstate(divide="ignore", invalid="ignore"):
                qx, qy = pr[:, 0] / z, pr[:, 1] / z
            front = z >= 0
            inside = front & (qx > -1) & (qx < W) & (qy > -1) & (qy < H)
            out_of_view += int((~inside).sum())
            near_edge += int((front & (((qx > -1) & (qx < 0)) | ((qy > -1) & (qy < 0)))).sum())
            if kinds[i] == "facade" and kinds[j] == "away":
                behind_away += int((z < 0).sum())
            if kinds[i] == "facade" and kinds[j] == "oblique":
                straddle += int(((z > 0).sum() > 0) and ((z < 0).sum() > 0))
    # partially overlapping views: some pairs inside, most outside, and
    # points landing within one pixel left of / above an image (column or
    # row 0 after truncation)
    assert 0.5 * total < out_of_view < total
    assert near_edge > 100
    # the views facing away have facade points behind them
    assert behind_away > 0.9 * sum(len(pts[i]) for i in range(n) if kinds[i] == "facade") * 2
    # the oblique view's camera plane cuts through facade surface of several views
    assert straddle >= 2
    assert (depths[kinds.index("oblique")] > 0).mean() > 0.5
    kept = sum(int((o > 0).sum()) for o in strip["ref"])
    assert kept > 0.05 * sum(int((d > 0).sum()) for d in depths)


def _removable_share(strip):
    """Share of the reference's (pixel, view) pairs that leave at the z or
    the bounds test (in float64: what a perfect per-pixel cull would skip)."""
    inv, ctw, KR, t = strip["mats"]
    depths = strip["depths"]
    n = len(depths)
    out, total = 0, 0
    for i, d in enumerate(depths):
        p = world_points(d, inv[i], ctw[i])
        for j in range(n):
            if j == i:
                continue
            pr = projections(p, KR[j], t[j])
            z = pr[:, 2]
            with np.errstate(divide="ignore", invalid="ignore"):
                qx, qy = pr[:, 0] / z, pr[:, 1] / z
            inside = (z >= 0) & (qx > -1) & (qx < W) & (qy > -1) & (qy < H)
            out += int((~inside).sum())
            total += len(pr)
    return out / total


@needs_oracle
@pytest.mark.gpu
def test_strip_scene_equal_and_culled(strip):
    got, st = api.cut_depth_maps(strip["depths"], strip["normals"], *strip["mats"],
                                 return_stats=True)
    _equal(got, strip["ref"])
    n = len(strip["depths"])
    valid = sum(int((d != 0).sum()) for d in strip["depths"])
    assert st["reference_pairs"] == valid * (n - 1)
    # a perfect per-pixel cull would drop `share` of the pairs; 16x16 tiles
    # whose box straddles an image border or the oblique camera's plane keep
    # some of them (about 1 % of the pairs here), so 80 % of the droppable
    # pairs must go
    share = _removable_share(strip)
    assert share > 0.8
    culled = 1.0 - st["evaluated_pairs"] / st["reference_pairs"]
    assert culled > 0.8 * share, (culled, share)
    assert st["target_groups"] == 1 and st["source_chunks"] >= 1
    assert st["ms_device"] > 0


@needs_oracle
@pytest.mark.gpu
def test_strip_scene_with_a_memory_cap(strip):
    """12 MB for 15 views of 1.9 MB each: several target groups, every source
    view streamed through one slot."""
    got, st = api.cut_depth_maps(strip["depths"], strip["normals"], *strip["mats"],
                                 device_bytes=12 << 20, return_stats=True)
    _equal(got, strip["ref"])
    assert st["target_groups"] >= 2 and st["source_chunks"] >= 3, st


@needs_oracle
@pytest.mark.gpu
def test_strip_scene_three_workers_on_one_device(strip):
    got, st = api.cut_depth_maps(strip["depths"], strip["normals"], *strip["mats"],
                                 devices=[0, 0, 0], return_stats=True)
    _equal(got, strip["ref"])
    assert st["target_groups"] >= 3


@needs_oracle
@pytest.mark.gpu
def test_strip_scene_two_devices(strip):
    if api.lib().smvsb_device_count() < 2:
        pytest.skip("needs two GPUs")
    L = api.lib()
    before = [L.smvsb_device_launch_count(d) for d in (0, 1)]
    got = api.cut_depth_maps(strip["depths"], strip["normals"], *strip["mats"], devices=[0, 1])
    _equal(got, strip["ref"])
    assert all(L.smvsb_device_launch_count(d) > b for d, b in zip((0, 1), before))


@needs_oracle
@pytest.mark.gpu
@pytest.mark.parametrize("device_bytes", [0, 8 << 20])
def test_ring_scene_through_the_multi_entry(device_bytes):
    """Five views around one object (test_gpu_cutmaps.make_views): every
    view sees every other, little is culled."""
    flen, rot, trans, depths, normals = make_views(5, W, H, 5)
    outs, inv, ctw, KR, t = oref.cut_depth_maps(flen, rot, trans, depths, normals)
    got, st = api.cut_depth_maps(depths, normals, inv, ctw, KR, t,
                                 device_bytes=device_bytes, return_stats=True)
    _equal(got, outs)
    assert st["evaluated_pairs"] > 0.5 * st["reference_pairs"]


@needs_oracle
@pytest.mark.gpu
@pytest.mark.skipif(not os.path.exists(oref.INTEGRATION_LIB_PATH),
                    reason="oracle/_ref/integration not built")
def test_strip_scene_through_the_drop_in_member(strip):
    flen, rot, trans, depths, normals, _ = strip_scene()
    gpu = oref.cut_depth_maps(flen, rot, trans, depths, normals,
                              lib_path=oref.INTEGRATION_LIB_PATH)[0]
    _equal(gpu, strip["ref"])


def _tiny_views(n=3):
    d = [np.full((8, 8), 2.0, np.float32) for _ in range(n)]
    nr = [np.zeros((8, 8, 3), np.float32) for _ in range(n)]
    eye = np.tile(np.eye(3, dtype=np.float32).reshape(9), (n, 1))
    ctw = np.tile(np.eye(4, dtype=np.float32).reshape(16), (n, 1))
    return d, nr, eye, ctw, eye.copy(), np.zeros((n, 3), np.float32)


def _call_multi(devices, device_bytes, views):
    d, nr, inv, ctw, KR, t = views
    n = len(d)
    outs = [np.empty_like(a) for a in d]
    w = (C.c_int * n)(*[8] * n)
    h = (C.c_int * n)(*[8] * n)
    dp = (C.c_void_p * n)(*[a.ctypes.data for a in d])
    npp = (C.c_void_p * n)(*[a.ctypes.data for a in nr])
    op = (C.c_void_p * n)(*[a.ctypes.data for a in outs])
    dv = (C.c_int * max(len(devices), 1))(*devices)
    opts = api.CutOptions(dv, len(devices), 0, device_bytes)
    L = api.lib()
    p = [a.ctypes.data_as(C.c_void_p) for a in (inv, ctw, KR, t)]
    rc = L.smvsb_cut_depth_maps_multi(C.byref(opts), n, w, h, dp, npp, *p, op, None)
    return rc, L.smvsb_last_error(None).decode()


@pytest.mark.gpu
@pytest.mark.parametrize("devices,device_bytes,message", [
    ([], 0, "empty device list"),
    ([0, 64], 0, "device index out of range"),
    ([-1], 0, "device index out of range"),
    ([0], 4096, "do not hold the largest target view and one source view"),
])
def test_multi_entry_rejects_bad_options(devices, device_bytes, message):
    rc, msg = _call_multi(devices, device_bytes, _tiny_views())
    assert rc == -1 and message in msg, (rc, msg)
    # the library is still usable afterwards
    rc, _ = _call_multi([0], 0, _tiny_views())
    assert rc == 0


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure path")
def test_multi_entry_without_gpu_has_no_cpu_fallback():
    rc, msg = _call_multi([0], 0, _tiny_views())
    assert rc == -2 and "no CPU fallback" in msg
    with pytest.raises(api.SmvsbError):
        api.cut_depth_maps(*_tiny_views(), devices=[0])
