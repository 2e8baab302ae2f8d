"""CPU side of tests/test_gpu_sgm_budget.py: the compiled reference's
SGMStereo::run_sgm on the 1920x1080 SGM scene of benchmarks/fullsize_cpu.py
at 32, 64, 128 and 256 planes (about 1 to 4 minutes each on one host core).
The depth maps are cached under benchmarks/_cache/ (git-ignored), keyed by
the plane count; the test starts this script, one process per missing plane
count, with its first test, so that the CPU work overlaps the GPU tests.

  python benchmarks/sgm_budget_cpu.py D [D ...]
"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "benchmarks")):
    if p not in sys.path:
        sys.path.insert(0, p)

CACHE = os.path.join(ROOT, "benchmarks", "_cache")
PLANES = (32, 64, 128, 256)
VERSION = 1           # bump when inputs change: old caches are then ignored


def cache_path(D):
    return os.path.join(CACHE, f"sgm_budget_v{VERSION}_1920x1080_seed9_D{D}.npz")


def run(D):
    import fullsize_cpu as fc
    from oracle import ref as oref
    t0 = time.time()
    sc, dmin, dmax = fc.sgm_scene()
    R = oref.RefScene(sc)
    try:
        depth = R.sgm_run(0, 1, 0, D, dmin, dmax)["depth"]
    finally:
        R.close()
    os.makedirs(CACHE, exist_ok=True)
    tmp = cache_path(D) + f".{os.getpid()}.tmp.npz"
    np.savez_compressed(tmp, depth=depth, seconds=time.time() - t0)
    os.replace(tmp, cache_path(D))
    print(f"D={D}: {time.time() - t0:.1f} s -> {cache_path(D)}")


if __name__ == "__main__":
    for d in sys.argv[1:] or PLANES:
        run(int(d))
