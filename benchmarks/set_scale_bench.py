"""StereoView::set_scale of 7 views (byte images up, scale 2 / 3 / 4) through
smvsb_set_views_u8, at one width on each side of the library's choice of
path: 1920 wide takes the TMA-engine staged fused kernel (cp.async.bulk +
mbarrier, one pass over the image); 1918 wide, whose rows are not a multiple
of 16 bytes, takes the three-kernel path (blur_x, blur_y, grad_hess, each a
round trip through L2/HBM). Prints one JSON line. The two paths' bitwise
agreement with the reference is checked by the GPU tests.

  python benchmarks/set_scale_bench.py [--reps 10]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from smvs_b200 import api  # noqa: E402
from smvs_b200.workload import build_workload  # noqa: E402

WIDTHS = {1920: "tma", 1918: "three_kernels"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    out = {"workload": "set_scale, 7 views x 1080 rows u8", "ms_per_call": {}}
    for scale in (2, 3, 4):
        for width, path in WIDTHS.items():
            wl = build_workload(width, 1080, 6, scale, shading=False, seed_index=0)
            with api.Context(0) as ctx:
                ts = []
                for _ in range(a.reps + 2):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    wl.push_views_u8(ctx)
                    torch.cuda.synchronize()
                    ts.append((time.perf_counter() - t0) * 1e3)
            out["ms_per_call"].setdefault(f"scale{scale}", {})[f"{path}_w{width}"] = \
                float(np.median(ts[2:]))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
