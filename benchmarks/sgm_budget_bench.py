"""SGM on the volume path against the banded path, in one process, alternating.

Sizes (128 planes, P1 = 6, P2 = 96, one main / neighbour pair; above 2 MP
the pair is a synthetic scene at half the size, upsampled 2 x 2):
  1920x1080   both paths fit; the banded run is capped at half the volume
              path's bytes, so this is the cost of banding;
  4800x3600   2.2e9 voxels: the volume path with an uncapped budget, the
              banded path under the default budget and under 4 GiB (partial
              sums staged through pinned host memory);
  9600x7200   8.8e9 voxels: only the banded path fits an 80 GB card.
For each run it prints one JSON line with the wall time (host clock around the
synchronous call, image upload and depth download included), the device time
(CUDA events), the bands, the peak device bytes and the host-staged bytes,
and whether the depth equals the other path's. The card's name and power
limit are read in the same run.

  python benchmarks/sgm_budget_bench.py [--reps N] [--sizes 1920x1080,4800x3600]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from smvs_b200 import api, synth  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                          "-i", "0"], capture_output=True, text=True).stdout.strip()
    return out or "unknown"


def pair(w, h):
    """A synthetic pair; above 2 MP a (w/2 x h/2) scene with each pixel repeated
    2 x 2 (the scene generator is slow at tens of megapixels) and the
    reprojection scaled to the doubled pixel coordinates."""
    f = 2 if w * h > 4e6 else 1
    sc = synth.make_scene(w // f, h // f, 1, seed_index=9)
    M, t = synth.reprojection(sc, 0)
    S = np.diag([float(f), float(f), 1.0])
    M = (S @ M.reshape(3, 3) @ np.linalg.inv(S)).astype(np.float32).ravel()
    t = (S @ t).astype(np.float32)
    imgs = [np.repeat(np.repeat(im, f, axis=0), f, axis=1) for im in sc.images[:2]]
    dmin, dmax = float(sc.true_depth.min() * 0.7), float(sc.true_depth.max() * 1.3)
    return imgs, M, t, dmin, dmax


def configs(w, h, D):
    """(label, device_bytes) of the runs at one size; 0 = the default budget."""
    volume = 10 * w * h * D
    if w * h <= 4e6:
        return [("volume", 0), ("banded", volume // 2)]
    if w * h <= 20e6:
        return [("volume", 60 << 30), ("banded", 0), ("banded_host", 4 << 30)]
    return [("banded", 0)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--planes", type=int, default=128)
    ap.add_argument("--sizes", default="1920x1080,4800x3600,9600x7200")
    a = ap.parse_args()
    gpu = card()
    for size in a.sizes.split(","):
        w, h = (int(x) for x in size.split("x"))
        (main, neigh), M, t, dmin, dmax = pair(w, h)
        runs = configs(w, h, a.planes)
        times = {label: [] for label, _ in runs}
        last = {}
        for rep in range(a.reps + 1):            # the first round warms up
            for label, budget in runs:
                t0 = time.perf_counter()
                r, st = api.sgm(main, neigh, M, t, dmin, dmax, a.planes,
                                device_bytes=budget, return_stats=True)
                wall = (time.perf_counter() - t0) * 1e3
                if rep > 0:
                    times[label].append((wall, st["ms_device"]))
                last[label] = (r["depth"], st)
        depths = [d for d, _ in last.values()]
        same = all(np.array_equal(depths[0], d) for d in depths[1:])
        for label, budget in runs:
            walls = sorted(x[0] for x in times[label])
            devs = sorted(x[1] for x in times[label])
            st = last[label][1]
            print(json.dumps({
                "size": f"{w}x{h}x{a.planes}", "path": label,
                "device_bytes": budget or "default", "gpu": gpu,
                "wall_ms_median": walls[len(walls) // 2], "wall_ms_all": walls,
                "device_ms_median": devs[len(devs) // 2],
                "banded": st["banded"], "bands": st["bands"],
                "peak_device_bytes": st["peak_device_bytes"],
                "host_bytes": st["host_bytes"],
                "depth_equal_across_paths": same,
                "valid_fraction": float((last[label][0] > 0).mean())}), flush=True)


if __name__ == "__main__":
    main()
