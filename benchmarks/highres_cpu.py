"""CPU side of tests/test_gpu_high_scales.py::test_ladder_from_scale_8: the
compiled reference's optimize() without SGM on a 6400x4300 colour scene
(3 neighbours, ladder 8 -> 7). It takes about 12 minutes on one host core, so
the result (the sparse initial depth and the depth map) is cached under
benchmarks/_cache/ (git-ignored), keyed by the scene parameters; the test
starts this script as a subprocess when the cache is missing, so that it
overlaps the module's other tests.

  python benchmarks/highres_cpu.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

CACHE = os.path.join(ROOT, "benchmarks", "_cache")
LADDER8 = dict(width=6400, height=4300, n_sub=3, seed=191, n_features=2000, min_scale=7)


def cache_path(job=LADDER8):
    return os.path.join(CACHE, "highres_nosgm_{width}x{height}_{n_sub}sub_seed{seed}"
                               "_f{n_features}_min{min_scale}.npz".format(**job))


def scene_and_features(job=LADDER8):
    from util_scene import colour_scene
    from test_gpu_topology import _features_on_surface
    sc = colour_scene(job["width"], job["height"], job["n_sub"], job["seed"])
    return sc, _features_on_surface(sc, job["n_features"], job["seed"])


def compute(job=LADDER8):
    from oracle import ref as oref
    sc, feats = scene_and_features(job)
    R = oref.RefScene(sc)
    try:
        sparse, depth, _ = R.optimize_nosgm(feats, regularization=0.01, num_iterations=5,
                                            min_scale=job["min_scale"])
    finally:
        R.close()
    os.makedirs(CACHE, exist_ok=True)
    tmp = cache_path(job) + f".{os.getpid()}.tmp.npz"
    np.savez(tmp, sparse=sparse, depth=depth)
    os.replace(tmp, cache_path(job))


if __name__ == "__main__":
    compute()
    print(cache_path())
