"""DepthOptimizer::optimize() resident on the device (smvsb_optimize_rgb_f32)
for views whose ladder starts at scale 7 or 8, without SGM: a seeded colour
view with 6 neighbours at 4000x3000 (12 MP, starts at scale 7) and at
6400x4300 (27.5 MP, starts at scale 8), down to min_scale 2.

Per scale of the ladder it prints the device time of each stage, summed from
the kernels of the CUDA activity trace of torch.profiler (the library's
stream is its own, so events on torch's stream would not bracket it):
set_scale, visibility, cutting, the Newton loops and the surface topology
between them. A scale starts with its set_scale kernels. Each size is run
once untimed, once timed and once under the profiler. The card's name and
power limit are read in the same run. Not part of the bench.py contract;
prints one JSON line per size.

  python benchmarks/highres_optimize.py [--sizes 4000x3000,6400x4300] [--out f]
"""
import argparse
import concurrent.futures
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from smvs_b200 import api, synth  # noqa: E402

N_SUB = 6
MIN_SCALE = 2
N_FEATURES = 4000

# kernel name -> stage; the first match wins
STAGES = (
    ("set_scale", ("blur_x_kernel", "blur_y_kernel", "grad_hess_kernel",
                   "set_scale_tma_kernel", "unpack_texels_kernel")),
    ("cutting", ("cut_depth_kernel", "cut_border_kernel")),
    ("visibility", ("zbuf_", "vis_patch", "vis_finalize", "vis_lists", "scan_kernel",
                    "render_kernel")),
    ("newton", ("gn_", "cg_", "reproj_kernel", "apply_delta", "update_reduce",
                "count_processed", "pack_subview")),
    ("topology", ("init_nodes", "fill_holes", "subdivide", "expand_", "remove_isolated",
                  "remove_nodes", "count_valid", "keep_positive")),
)


def stage_of(name):
    for stage, keys in STAGES:
        if any(k in name for k in keys):
            return stage
    return "other"


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return None


def colour_view(width, height, seed):
    """synth.make_scene with three different channels per view, as float RGB
    in [0, 1] (StereoView::get_image() of a colour view), the poses, and a
    sparse depth of N_FEATURES surface points (what Surface::create projects
    from a bundle)."""
    sc = synth.make_scene(width, height, N_SUB, seed_index=seed)
    rng = np.random.default_rng(seed)
    gains = ((1.0, 0.0), (0.8, 20.0), (1.1, -10.0))
    noise_seeds = rng.integers(0, 2**31, size=len(sc.images))

    def to_rgb(k):
        f = sc.images[k].astype(np.float32)
        r = np.random.default_rng(int(noise_seeds[k]))
        ch = [np.clip(f * g + o + r.normal(0, 2.0, f.shape), 0, 255).astype(np.uint8)
              for g, o in gains]
        return np.stack(ch, axis=2).astype(np.float32) / np.float32(255)

    with concurrent.futures.ThreadPoolExecutor(max_workers=8) as ex:
        images = list(ex.map(to_rgb, range(len(sc.images))))
    Mt = [synth.reprojection(sc, k) for k in range(N_SUB)]
    Mi = np.array([m for m, _ in Mt], dtype=np.float64).reshape(N_SUB, 9)
    ti = np.array([t for _, t in Mt], dtype=np.float64).reshape(N_SUB, 3)
    ax = np.float32(sc.flen[0]) * np.float32(max(width, height))
    K = np.array([1 / ax, 0, -np.float32(width) * np.float32(0.5) / ax,
                  0, 1 / ax, -np.float32(height) * np.float32(0.5) / ax, 0, 0, 1],
                 dtype=np.float32)
    sparse = np.zeros((height, width), np.float32)
    x = rng.integers(8, width - 8, N_FEATURES)
    y = rng.integers(8, height - 8, N_FEATURES)
    sparse[y, x] = sc.true_depth[y, x]
    return images, Mi, ti, float(ax), float(np.float32(1.0) / ax), K, sparse


def run(ctx, view):
    images, Mi, ti, flen_px, inv_flen, K, sparse = view
    return api.optimize(ctx, images[0], images[1:], Mi, ti, flen_px, inv_flen, K, sparse,
                        num_iterations=5, min_scale=MIN_SCALE, use_sgm=False)


def per_scale(events, start_scale):
    """Device ms per stage and scale; a scale begins at a set_scale kernel
    that follows kernels of another stage."""
    kernels = sorted((e for e in events if e.device_type == torch.autograd.DeviceType.CUDA
                      and e.time_range.elapsed_us() >= 0),
                     key=lambda e: e.time_range.start)
    scales, cur, prev = [], None, None
    for e in kernels:
        st = stage_of(e.name)
        if st == "set_scale" and prev != "set_scale":
            cur = {}
            scales.append(cur)
        if cur is not None:
            cur[st] = cur.get(st, 0.0) + e.time_range.elapsed_us() / 1e3
        prev = st
    return [dict(scale=start_scale - i, **{k: round(v, 3) for k, v in s.items()})
            for i, s in enumerate(scales)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="4000x3000,6400x4300")
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("highres_optimize.py: no CUDA device")
    device, limit = torch.cuda.get_device_name(0), power_limit()
    lines = []
    with api.Context(0) as ctx:
        for size in a.sizes.split(","):
            w, h = (int(v) for v in size.split("x"))
            view = colour_view(w, h, 7)
            # an untimed run of the same view first: every kernel its ladder
            # uses is loaded and every buffer allocated before the timed runs
            run(ctx, view)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            d, _, _, st = run(ctx, view)
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) * 1e3
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                d2, _, _, _ = run(ctx, view)
                torch.cuda.synchronize()
            start = st["final_scale"] + st["scales"] - 1
            rows = per_scale(prof.events(), start)
            out = {"device": device, "power_limit": limit,
                   "workload": f"optimize() {w}x{h} colour, {N_SUB} neighbours, no SGM, "
                               f"scales {start}..{st['final_scale']}",
                   "ms_wall": round(wall, 1), "valid_fraction": float((d > 0).mean()),
                   "repeat_identical": bool(np.array_equal(d, d2)), "stats": st,
                   "device_ms_per_scale": rows}
            lines.append(json.dumps(out))
            print(lines[-1], flush=True)
    if a.out:
        with open(a.out, "a") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
