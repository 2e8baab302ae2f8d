"""MeshGenerator::cut_depth_maps on scenes of many 1920x1080 views. Not part of
the bench.py contract; prints one JSON line per scene and run, then a summary.

Scenes (seeded, closed-form geometry, matrices from the compiled reference's
camera code via oracle.ref.cut_depth_maps(..., run=False)):
  seven  the 7-view case of tests/test_gpu_cutmaps.py (BASELINE.json's size)
  ring   48 views on a circle, all looking at one height field
         (tests/test_gpu_cut_scene.ring_scene): every view sees every other
  strip  160 views along a facade (tests/test_gpu_cut_scene.strip_scene):
         each view overlaps a few neighbours, culling dominates
Runs per scene, alternated rep by rep in one process after one warm-up each:
  old     smvsb_cut_depth_maps on device 0
  base    smvsb_cut_depth_maps of another build (--baseline-lib), e.g. the
          parent commit's library: before / after in one session
  new1    smvsb_cut_depth_maps_multi, devices [0]
  all     smvsb_cut_depth_maps_multi, every device (only with >= 2 GPUs)
  capped  smvsb_cut_depth_maps_multi, devices [0], a cap that forces >= 4
          source chunks
Every run's maps are compared with the first run's (np.array_equal).

  python benchmarks/cut_scene_bench.py [--scenes seven,ring,strip] [--reps 3]
                                       [--baseline-lib PATH]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from smvs_b200 import api  # noqa: E402
from oracle import ref as oref  # noqa: E402
from test_gpu_cutmaps import make_views  # noqa: E402
from test_gpu_cut_scene import ring_scene, strip_scene  # noqa: E402

W, H = 1920, 1080


def make_scene(name):
    if name == "seven":
        flen, rot, trans, depths, normals = make_views(7, W, H, 7)
    elif name == "ring":
        flen, rot, trans, depths, normals, _ = ring_scene(48, W, H, 48, iters=6)
    else:
        flen, rot, trans, depths, normals, _ = strip_scene(seed=160, n_facade=157, w=W, h=H,
                                                            iters=6)
    _, inv, ctw, KR, t = oref.cut_depth_maps(flen, rot, trans, depths, normals, run=False)
    return depths, normals, (inv, ctw, KR, t)


def call_lib(L, depths, normals, mats, device=0):
    """smvsb_cut_depth_maps of library L (loaded by path)."""
    n = len(depths)
    outs = [np.empty_like(a) for a in depths]
    w = (C.c_int * n)(*[a.shape[1] for a in depths])
    h = (C.c_int * n)(*[a.shape[0] for a in depths])
    dp = (C.c_void_p * n)(*[a.ctypes.data for a in depths])
    npp = (C.c_void_p * n)(*[a.ctypes.data for a in normals])
    op = (C.c_void_p * n)(*[a.ctypes.data for a in outs])
    m = [np.ascontiguousarray(a, np.float32).reshape(-1).ctypes.data_as(C.c_void_p)
         for a in mats]
    rc = L.smvsb_cut_depth_maps(device, n, w, h, dp, npp, *m, op)
    if rc != 0:
        L.smvsb_last_error.restype = C.c_char_p
        raise RuntimeError(L.smvsb_last_error(None).decode())
    return outs


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit",
                               "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip().splitlines()
    except (OSError, subprocess.SubprocessError):
        return ["not available"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="seven,ring,strip")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--baseline-lib", default=None)
    a = ap.parse_args()
    n_dev = api.lib().smvsb_device_count()
    if n_dev < 1:
        sys.exit("no CUDA device: nothing measured")
    base = C.CDLL(os.path.abspath(a.baseline_lib)) if a.baseline_lib else None
    print(json.dumps({"gpus": gpu_info(), "device_count": n_dev}), flush=True)
    summary = {}
    for name in a.scenes.split(","):
        t0 = time.perf_counter()
        depths, normals, mats = make_scene(name)
        gen_s = time.perf_counter() - t0
        pix = sum(d.size for d in depths)
        # about 25 bytes per target pixel: a quarter of the scene per group
        cap = max(25 * pix // 4, 200 << 20)
        runs = {"old": lambda: (api.cut_depth_maps(depths, normals, *mats), None),
                "new1": lambda: api.cut_depth_maps(depths, normals, *mats, devices=[0],
                                                   return_stats=True),
                "capped": lambda: api.cut_depth_maps(depths, normals, *mats, devices=[0],
                                                     device_bytes=cap, return_stats=True)}
        if base is not None:
            runs["base"] = lambda: (call_lib(base, depths, normals, mats), None)
        if n_dev > 1:
            runs["all"] = lambda: api.cut_depth_maps(depths, normals, *mats,
                                                     devices=list(range(n_dev)),
                                                     return_stats=True)
        first, stats, times = None, {}, {k: [] for k in runs}
        for rep in range(a.reps + 1):            # rep 0 warms up every run
            for k, fn in runs.items():
                t0 = time.perf_counter()
                outs, st = fn()
                dt = time.perf_counter() - t0
                if first is None:
                    first = outs
                elif not all(np.array_equal(x, y) for x, y in zip(outs, first)):
                    raise SystemExit(f"{name}/{k}: maps differ from the first run")
                if rep > 0:
                    times[k].append(dt)
                if st is not None:
                    stats[k] = st
        res = {"scene": name, "views": len(depths), "size": f"{W}x{H}",
               "generate_s": round(gen_s, 1), "equal": True,
               "seconds": {k: {"mean": float(np.mean(v)), "min": float(np.min(v)),
                               "max": float(np.max(v))} for k, v in times.items()},
               "stats": stats, "cap_bytes": int(cap)}
        print(json.dumps(res), flush=True)
        summary[name] = {k: round(float(np.mean(v)), 4) for k, v in times.items()}
        del depths, normals, first
    print(json.dumps({"summary_mean_seconds": summary, "gpus": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
