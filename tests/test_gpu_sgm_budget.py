"""SGM within a device-memory budget (smvsb_sgm_ex, smvsb_sgm_reconstruct_ex).

When the cost and aggregation volumes of a run (about 10 bytes per voxel) do
not fit the budget, run_sgm runs in bands of image rows: cost per band, a
top-to-bottom sweep that keeps uint16 partial sums (on the device, or staged
through pinned host memory), and a bottom-to-top sweep that adds them and takes
the winner. The depth must be bit-identical to the compiled reference's
(oracle/_ref) whatever the budget:
  * 1920x1080 at 32, 64, 128 and 256 planes with 2 bands, many bands and
    host-staged partial sums (the reference runs in subprocesses started with
    the first test, benchmarks/sgm_budget_cpu.py, cached under
    benchmarks/_cache/);
  * bands of 16 rows (every boundary inside the census halo), an odd height,
    and an image narrower than a band (the diagonals wrap around inside bands
    and across band boundaries);
  * reconstruct and the two-neighbour merge under a banding budget;
  * 4800x3600x128 (2.2e9 voxels): banded under the default budget against the
    volume path with an uncapped budget, in one process;
  * the error paths: a budget below the minimum names the minimum; without a
    GPU the call fails with SMVSB_ERR_CUDA.
Then SGM as smvsrecon runs it followed by optimize() in SGM mode from scale 7
(6400x4300) and from scale 8 (12800x8600, 110 MP, banded SGM, on one card),
against the scene's ground truth.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from smvs_b200 import api, synth
from oracle import ref as oref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
import fullsize_cpu as fc  # noqa: E402
import sgm_budget_cpu as sbc  # noqa: E402


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:
        return False


needs_ref = pytest.mark.skipif(not oref.available(), reason="oracle/_ref not built")


# -- the workspace sizes of sgm.cu (pair_plan, Fixed), to aim budgets at a band
# height; the tests check the outcome through the returned stats ------------

def volume_bytes(w, h, D, rows, host):
    """Device bytes of one banded run besides the images and depth maps."""
    pitch = (w + 63) // 64 * 64 + 16
    cost = w * D * rows
    warp = pitch * ((rows + 15) // 16 * 16 + 6) * D
    part = (2 * cost if host else w * h * D) * 2
    state = 6 * w * (D // 8) * 16
    return 6 * cost + warp + part + state


def run_fixed_bytes(w, h):
    """Images, the neighbour's float copy, the depth map and the plane depths
    of smvsb_sgm_ex with a main and a neighbour of the same size."""
    return 2 * w * h + (2 * w * h + 512) * 4


def reconstruct_fixed_bytes(w, h, merge):
    return 2 * w * h + ((4 + merge) * w * h + 512) * 4


def budget_for(w, h, D, rows, host):
    return run_fixed_bytes(w, h) + volume_bytes(w, h, D, rows, host)


def expected_bands(w, h, D, avail):
    """(band rows, host staging) sgm.cu chooses for `avail` volume bytes: the
    tallest bands (multiples of 16 rows) that fit, partial sums on the device
    unless that leaves bands under min(64, the host-staged height)."""
    def most(host):
        for r in range((h + 15) // 16 * 16, 15, -16):
            if volume_bytes(w, h, D, r, host) <= avail:
                return r
        return 0
    on_device, on_host = most(False), most(True)
    if on_device > 0 and on_device >= min(on_host, 64):
        return on_device, False
    return on_host, True


@pytest.fixture(scope="module")
def ref_1080():
    """The reference's 1920x1080 depth per plane count: from benchmarks/_cache/
    when present, otherwise computed in one subprocess per plane count, started
    with the module's first test."""
    procs = {}
    if oref.available() and _has_gpu():
        for D in sbc.PLANES:
            if not os.path.exists(sbc.cache_path(D)):
                procs[D] = subprocess.Popen(
                    [sys.executable, os.path.join(ROOT, "benchmarks", "sgm_budget_cpu.py"),
                     str(D)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)

    def get(D):
        p = procs.pop(D, None)
        if p is not None:
            out, _ = p.communicate(timeout=1800)
            assert p.returncode == 0, out[-2000:]
        return np.load(sbc.cache_path(D))["depth"]

    yield get
    for p in procs.values():
        p.kill()
        p.wait()


@pytest.fixture(scope="module")
def inputs_1080():
    return fc.sgm_inputs()


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("D", [32, 64, 128, 256])
def test_banded_1080p_matches_reference(ref_1080, inputs_1080, D):
    """Two bands, seventeen bands of 64 rows (partial sums on the device) and
    nine bands of 128 rows with the partial sums staged through the host."""
    sc, dmin, dmax, M, t = inputs_1080
    w, h = 1920, 1080
    runs = [(544, False, 2), (64, False, 17), (128, True, 9)]
    outs = []
    for rows, host, bands in runs:
        budget = budget_for(w, h, D, rows, host)
        r, st = api.sgm(sc.images[0], sc.images[1], M, t, dmin, dmax, D,
                        device_bytes=budget, return_stats=True)
        assert st["banded"] == 1 and st["bands"] == bands, (rows, host, st)
        assert (st["host_bytes"] == w * h * D * 2) == host, st
        assert st["host_bytes"] in (0, w * h * D * 2), st
        assert st["peak_device_bytes"] <= budget, st
        outs.append(r["depth"])
    ref = ref_1080(D)
    for (rows, host, _), d in zip(runs, outs):
        assert np.array_equal(d, ref), (D, rows, host)


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("w,h,D,rows", [
    (333, 207, 64, 16),      # odd height, 13 bands: every boundary in the census halo
    (333, 207, 64, 48),
    (40, 301, 32, 16),       # narrower than a band: diagonals wrap inside bands
    (40, 301, 32, 64),       # and across their boundaries
    (200, 150, 256, 32),
    (97, 1001, 128, 80),
])
@pytest.mark.parametrize("host", [False, True])
def test_banded_small_matches_reference(w, h, D, rows, host):
    sc = synth.make_scene(w, h, 1, seed_index=9)
    R = oref.RefScene(sc)
    dmin, dmax = float(sc.true_depth.min() * 0.7), float(sc.true_depth.max() * 1.3)
    ref = R.sgm_run(0, 1, 0, D, dmin, dmax)["depth"]
    M, t = R.reprojection(0, 1, w, h, w, h)
    R.close()
    budget = budget_for(w, h, D, rows, host)
    r, st = api.sgm(sc.images[0], sc.images[1], M, t, dmin, dmax, D,
                    device_bytes=budget, return_stats=True)
    band_rows, staged = expected_bands(w, h, D, volume_bytes(w, h, D, rows, host))
    assert st["banded"] == 1 and st["bands"] == -(-h // band_rows), (band_rows, st)
    assert st["host_bytes"] == (w * h * D * 2 if staged else 0), st
    assert st["peak_device_bytes"] <= budget, st
    assert np.array_equal(r["depth"], ref)
    g = api.sgm(sc.images[0], sc.images[1], M, t, dmin, dmax, D)
    assert np.array_equal(g["depth"], ref)


@pytest.mark.gpu
@needs_ref
def test_banded_reconstruct_and_merge_match_reference():
    """smvsb_sgm_reconstruct_ex with both runs banded (partial sums on the
    device, then staged through the host), with and without merge_with,
    against SGMStereo::reconstruct and the merge of app/smvsrecon.cc:362-377."""
    w, h, D = 352, 264, 64
    sc = synth.make_scene(w, h, 2, seed_index=23)
    dmin, dmax = float(sc.true_depth.min() * 0.7), float(sc.true_depth.max() * 1.3)
    R = oref.RefScene(sc)
    ref = [R.sgm_reconstruct(0, k, 0, D, dmin, dmax) for k in (1, 2)]
    mats = [(R.reprojection(0, k, w, h, w, h), R.reprojection(k, 0, w, h, w, h))
            for k in (1, 2)]
    R.close()
    d1, d2 = ref[0].copy(), ref[1]
    both = (d1 != 0) & (d2 != 0)
    only2 = (d1 == 0) & (d2 != 0)
    d1[both] = (d1[both] + d2[both]) * np.float32(0.5)
    d1[only2] = d2[only2]
    for rows, host in ((80, False), (48, True)):
        prev = None
        for k in (1, 2):
            (M_mn, t_mn), (M_nm, t_nm) = mats[k - 1]
            budget = reconstruct_fixed_bytes(w, h, prev is not None) \
                + volume_bytes(w, h, D, rows, host)
            single, st = api.sgm_reconstruct(
                sc.images[0], sc.images[k], M_mn, t_mn, M_nm, t_nm, (dmin, dmax),
                (dmin, dmax), D, device_bytes=budget, return_stats=True)
            band_rows, staged = expected_bands(w, h, D, volume_bytes(w, h, D, rows, host))
            assert staged == host
            assert st["banded"] == 1 and st["bands"] == -(-h // band_rows), st
            assert st["host_bytes"] == (2 * w * h * D * 2 if staged else 0), st
            assert st["peak_device_bytes"] <= budget, st
            assert np.array_equal(single["depth"], ref[k - 1])
            out, st = api.sgm_reconstruct(
                sc.images[0], sc.images[k], M_mn, t_mn, M_nm, t_nm, (dmin, dmax),
                (dmin, dmax), D, merge_with=prev,
                device_bytes=reconstruct_fixed_bytes(w, h, True)
                + volume_bytes(w, h, D, rows, host), return_stats=True)
            assert st["banded"] == 1
            prev = out["depth"]
        assert np.array_equal(prev, d1), (rows, host)


def doubled_pair(w, h, seed_index=9):
    """A 2w x 2h pair: each pixel of a synthetic w x h scene repeated 2 x 2,
    the reprojection scaled to the doubled pixel coordinates."""
    sc = synth.make_scene(w, h, 1, seed_index=seed_index)
    M, t = synth.reprojection(sc, 0)
    S = np.diag([2.0, 2.0, 1.0])
    M2 = (S @ M.reshape(3, 3) @ np.linalg.inv(S)).astype(np.float32).ravel()
    t2 = (S @ t).astype(np.float32)
    up = [np.repeat(np.repeat(im, 2, axis=0), 2, axis=1) for im in sc.images[:2]]
    dmin, dmax = float(sc.true_depth.min() * 0.7), float(sc.true_depth.max() * 1.3)
    return up, M2, t2, dmin, dmax


@pytest.mark.gpu
def test_past_2_31_voxels_banded_equals_volume_path():
    """4800x3600x128 = 2.2e9 voxels: about 22 GB of volumes, more than the
    default budget of a quarter of an 80 GB card, so the default call takes
    the banded path. Under 8 GiB it runs in several bands with the partial
    sums on the device, under 4 GiB with them staged through the host. The
    volume path with an uncapped budget gives the same depth, bitwise."""
    w, h, D = 4800, 3600, 128
    (main, neigh), M, t, dmin, dmax = doubled_pair(w // 2, h // 2)
    whole, sw = api.sgm(main, neigh, M, t, dmin, dmax, D, device_bytes=60 << 30,
                        return_stats=True)
    assert sw["banded"] == 0 and sw["bands"] == 1, sw
    assert sw["peak_device_bytes"] > 10 * w * h * D, sw
    assert 0.3 < (whole["depth"] > 0).mean()
    quarter = _card_bytes() // 4
    for budget, staged in ((0, None), (8 << 30, False), (4 << 30, True)):
        banded, sb = api.sgm(main, neigh, M, t, dmin, dmax, D, device_bytes=budget,
                             return_stats=True)
        assert sb["banded"] == 1, (budget, sb)
        if staged is None:
            # the workspace held the volume path's 22 GB; the default call
            # gives back what its budget does not hold
            assert sb["peak_device_bytes"] <= quarter, sb
        else:
            assert sb["bands"] > 1 and sb["peak_device_bytes"] <= budget, sb
            assert sb["host_bytes"] == (w * h * D * 2 if staged else 0), sb
        assert np.array_equal(banded["depth"], whole["depth"]), budget


def _card_bytes():
    import torch
    return torch.cuda.get_device_properties(0).total_memory


@pytest.mark.gpu
@needs_ref
def test_volume_path_unchanged_within_budget(inputs_1080):
    """Inside the budget the call is the volume path, with its 5 launches per
    run_sgm; the volume dumps take it whatever the budget."""
    sc, dmin, dmax, M, t = inputs_1080
    r, st = api.sgm(sc.images[0], sc.images[1], M, t, dmin, dmax, 128, return_stats=True)
    assert st["banded"] == 0 and st["bands"] == 1 and st["host_bytes"] == 0, st
    assert st["ms_device"] > 0
    n0 = api.lib().smvsb_device_launch_count(0)
    api.sgm(sc.images[0], sc.images[1], M, t, dmin, dmax, 128, device_bytes=8 << 30)
    assert api.lib().smvsb_device_launch_count(0) - n0 == 5
    # dumps always take the volume path, whatever the budget
    v, sv = api.sgm(sc.images[0][:200, :300], sc.images[1][:200, :300], M, t, dmin, dmax,
                    64, volumes=True, device_bytes=8 << 20, return_stats=True)
    assert sv["banded"] == 0 and v["sgm"] is not None


@pytest.mark.gpu
def test_budget_below_minimum_names_it():
    w, h, D = 640, 480, 128
    sc = synth.make_scene(w, h, 1, seed_index=9)
    M, t = np.eye(3, dtype=np.float32).ravel(), np.zeros(3, np.float32)
    minimum = budget_for(w, h, D, 16, True)
    with pytest.raises(api.SmvsbError) as e:
        api.sgm(sc.images[0], sc.images[1], M, t, 1.0, 2.0, D, device_bytes=minimum - 1)
    assert e.value.code == -1
    assert f"minimum of {minimum} bytes" in str(e.value)
    _, st = api.sgm(sc.images[0], sc.images[1], M, t, 1.0, 2.0, D,
                    device_bytes=minimum, return_stats=True)
    assert st["banded"] == 1 and st["bands"] == h // 16 and st["host_bytes"] > 0, st
    assert st["peak_device_bytes"] <= minimum
    with pytest.raises(api.SmvsbError) as e:
        api.sgm_reconstruct(sc.images[0], sc.images[1], M, t, M, t, (1.0, 2.0), (1.0, 2.0),
                            D, device_bytes=1 << 20)
    assert e.value.code == -1 and "minimum of" in str(e.value)


@pytest.mark.skipif(_has_gpu(), reason="checks the no-GPU failure path")
def test_ex_entry_points_without_gpu():
    """Without a device both entry points fail with SMVSB_ERR_CUDA (-2) and
    say that there is no CPU fallback; NULL options and stats are accepted."""
    L = api.lib()
    z = np.zeros((64, 64), np.uint8)
    eye, t0 = np.eye(3, dtype=np.float32).ravel(), np.zeros(3, np.float32)
    depth = np.empty((64, 64), np.float32)
    rng = np.array([1.0, 2.0], np.float32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)  # noqa: E731
    for opts in (None, C.byref(api.SgmOptions(1 << 30))):
        st = api.SgmStats()
        rc = L.smvsb_sgm_ex(0, 64, 64, p(z), 64, 64, p(z), p(eye), p(t0), C.c_float(1.0),
                            C.c_float(2.0), 64, C.c_uint16(6), C.c_uint16(96), p(depth),
                            None, None, None, opts, C.byref(st))
        assert rc == -2 and b"no CPU fallback" in L.smvsb_last_error(None)
        rc = L.smvsb_sgm_reconstruct_ex(0, 64, 64, p(z), 64, 64, p(z), p(eye), p(t0), p(eye),
                                        p(t0), p(rng), p(rng), 64, C.c_uint16(6),
                                        C.c_uint16(96), None, p(depth), None, opts, None)
        assert rc == -2 and b"no CPU fallback" in L.smvsb_last_error(None)
    with pytest.raises(api.SmvsbError) as e:
        api.sgm(z, z, eye, t0, 1.0, 2.0, 64, device_bytes=1 << 30)
    assert e.value.code == -2
    # the reserved option fields are checked with the arguments
    bad = api.SgmOptions(1 << 30)
    bad.reserved[1] = 7
    rc = L.smvsb_sgm_ex(0, 64, 64, p(z), 64, 64, p(z), p(eye), p(t0), C.c_float(1.0),
                        C.c_float(2.0), 64, C.c_uint16(6), C.c_uint16(96), p(depth),
                        None, None, None, C.byref(bad), None)
    assert rc == -1 and b"reserved" in L.smvsb_last_error(None)


# -- optimize() in SGM mode from scales 7 and 8, after the device SGM ---------
#
# A 3200x2150 synthetic scene with 3 neighbours, its pixels repeated f x f:
# f = 2 gives 6400x4300 (27.5 MP, the SGM ladder starts at scale 7), f = 4
# 12800x8600 (110 MP, starts at scale 8). As smvsrecon does by default, SGM
# runs on half-size images against two neighbours (reconstruct, then the merge
# of the second result into the first), and optimize() starts from it.

BASE_W, BASE_H, N_SUB = 3200, 2150, 3


@pytest.fixture(scope="module")
def ladder_scene():
    return synth.make_scene(BASE_W, BASE_H, N_SUB, seed_index=193)


def _repeat(a, f):
    return np.repeat(np.repeat(a, f, axis=0), f, axis=1) if f > 1 else a


def _calib(sc, v, w, h):
    ax = float(sc.flen[v]) * max(w, h)
    return np.array([[ax, 0, w * 0.5], [0, ax, h * 0.5], [0, 0, 1]])


def _reprojection(sc, a, b, w, h):
    """M, t of view a's pixels to view b at w x h (fill_reprojection)."""
    Ra, Rb = sc.rot[a].reshape(3, 3), sc.rot[b].reshape(3, 3)
    Ka, Kb = _calib(sc, a, w, h), _calib(sc, b, w, h)
    M = Kb @ Rb @ Ra.T @ np.linalg.inv(Ka)
    t = Kb @ (sc.trans[b] - Rb @ Ra.T @ sc.trans[a])
    return M.astype(np.float32).ravel(), t.astype(np.float32)


def _sgm_then_optimize(sc, f, min_scale):
    w, h = BASE_W * f, BASE_H * f
    sw, sh = w // 2, h // 2
    sgm_imgs = [_repeat(im, f // 2) for im in sc.images]
    rng = (float(sc.true_depth.min() * 0.7), float(sc.true_depth.max() * 1.3))
    depth, sgm_stats = None, []
    for k in (1, 2):
        M_mn, t_mn = _reprojection(sc, 0, k, sw, sh)
        M_nm, t_nm = _reprojection(sc, k, 0, sw, sh)
        r, st = api.sgm_reconstruct(sgm_imgs[0], sgm_imgs[k], M_mn, t_mn, M_nm, t_nm, rng,
                                    rng, 128, merge_with=depth, return_stats=True)
        depth = r["depth"]
        sgm_stats.append(st)
    del sgm_imgs
    imgs = [_repeat(im, f) for im in sc.images]
    Mt = [_reprojection(sc, 0, k, w, h) for k in range(1, N_SUB + 1)]
    Mi = np.array([m for m, _ in Mt], np.float64).reshape(N_SUB, 9)
    ti = np.array([t for _, t in Mt], np.float64).reshape(N_SUB, 3)
    K = _calib(sc, 0, w, h)
    Ki = np.linalg.inv(K).astype(np.float32).ravel()
    import torch
    with api.Context(0) as ctx:
        d, _, _, st = api.optimize(ctx, imgs[0], imgs[1:], Mi, ti, K[0, 0], 1.0 / K[0, 0], Ki,
                                   depth, min_scale=min_scale, use_sgm=True)
        free, total = torch.cuda.mem_get_info(0)
    truth = _repeat(sc.true_depth, f)
    m = d > 0
    rel = np.abs(d[m] - truth[m]) / truth[m]
    out = dict(sgm=sgm_stats, optimize=st, valid=float(m.mean()),
               sgm_valid=float((depth > 0).mean()), rel_median=float(np.median(rel)),
               rel_p90=float(np.percentile(rel, 90)), device_used_after=total - free)
    print(out)
    return out


@pytest.mark.gpu
def test_sgm_ladder_from_scale_7(ladder_scene):
    """6400x4300: the SGM images (3200x2150x128) take the volume path under the
    default budget; optimize() in SGM mode starts at scale 7 and runs to 6."""
    r = _sgm_then_optimize(ladder_scene, 2, 6)
    assert all(s["banded"] == 0 for s in r["sgm"]), r["sgm"]
    assert r["optimize"]["final_scale"] == 6 and r["optimize"]["scales"] == 2, r["optimize"]
    assert r["sgm_valid"] > 0.3 and r["valid"] > 0.5, r
    assert r["rel_median"] < 5e-4 and r["rel_p90"] < 2e-3, r


@pytest.mark.gpu
def test_sgm_ladder_from_scale_8_fits_one_gpu(ladder_scene):
    """12800x8600 (110 MP): its SGM images (6400x4300x128, 3.5e9 voxels, about
    35 GB on the volume path) take the banded path under the default budget,
    and optimize() in SGM mode from scale 8 to 7 completes next to the SGM
    workspace on one card, within the depth error of the scale-7 run."""
    r = _sgm_then_optimize(ladder_scene, 4, 7)
    assert all(s["banded"] == 1 and s["bands"] >= 1 for s in r["sgm"]), r["sgm"]
    assert all(s["peak_device_bytes"] <= _card_bytes() // 4 for s in r["sgm"]), r["sgm"]
    assert r["optimize"]["final_scale"] == 7 and r["optimize"]["scales"] == 2, r["optimize"]
    assert r["sgm_valid"] > 0.3 and r["valid"] > 0.5, r
    assert r["rel_median"] < 5e-4 and r["rel_p90"] < 2e-3, r
