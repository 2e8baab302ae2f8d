"""The PCG solves of one bench.py view (1920x1080, scale 2, no shading), one
Newton step at a time through the ABI calls (gn_construct -> cg_solve ->
update_nodes, the loop of smvsb_newton_loop), to show where the solve's time
goes as the system shrinks. Per Newton step: block rows and 4x4 blocks of the
system, CG iterations, and microseconds per iteration of cg_kernel (device
time of the kernel from the CUDA activity trace of torch.profiler; the
library's stream is its own, so events recorded on torch's stream would not
bracket it) and of the whole cg_solve call (host clock; the call ends in a
stream synchronise and includes the row-list kernels and the launch). Ends with
one JSON line that also names the device and its power limit. Not part of the
bench.py contract.

  python benchmarks/cg_bench.py [--view 0] [--out FILE]
"""
import argparse
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
from smvs_b200 import api  # noqa: E402
from smvs_b200.workload import build_workload  # noqa: E402

REGULARIZATION = 0.01


def system_size(wl, active):
    """(block rows, 4x4 blocks) of the system over the nodes that are valid
    and active: a block exists where both of its nodes are."""
    on = (wl.node_valid.astype(bool) & active.astype(bool)).reshape(wl.npy + 1, wl.npx + 1)
    blocks = 0
    for dy in (-1, 0, 1):
        for dx in (-1, 0, 1):
            a = on[max(dy, 0):on.shape[0] + min(dy, 0), max(dx, 0):on.shape[1] + min(dx, 0)]
            b = on[max(-dy, 0):on.shape[0] + min(-dy, 0), max(-dx, 0):on.shape[1] + min(-dx, 0)]
            blocks += int((a & b).sum())
    return int(on.sum()), blocks


def newton_loop(ctx, wl):
    """One inner Newton loop; per step (rows, blocks, iterations, solve wall s)."""
    ctx.set_nodes(wl.nodes)
    n_initial = int(wl.node_valid.astype(bool).sum())
    active, n_active, steps = None, n_initial, []
    while n_active > n_initial // 20 and len(steps) < 200:
        rows, blocks = system_size(wl, wl.node_valid if active is None else active)
        ctx.gn_construct(active, None, REGULARIZATION, 0.0)
        t0 = time.perf_counter()
        iters, _ = ctx.cg_solve()
        wall = time.perf_counter() - t0
        active, n_active, _ = ctx.update_nodes()
        steps.append((rows, blocks, iters, wall))
    return steps


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                               "-i", "0"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--view", type=int, default=0, help="seed of the bench.py pool view")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("cg_bench.py: no CUDA device")
    wl = build_workload(1920, 1080, 6, 2, shading=False, seed_index=a.view)
    with api.Context(0) as ctx:
        wl.push_views_u8(ctx)
        wl.push_surface(ctx)
        newton_loop(ctx, wl)                         # warm-up
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            steps = newton_loop(ctx, wl)
        kernels = sorted((e for e in prof.events() if "cg_kernel" in e.name),
                         key=lambda e: e.time_range.start)
        ctx.set_nodes(wl.nodes)
        st = ctx.newton_loop(None, REGULARIZATION, 0.0)
    if len(kernels) != len(steps):
        raise SystemExit(f"cg_bench.py: {len(kernels)} cg_kernel launches traced "
                         f"for {len(steps)} Newton steps")
    if (st["newton_steps"], st["cg_iterations"]) != (len(steps), sum(s[2] for s in steps)):
        raise SystemExit("cg_bench.py: the stepped loop differs from smvsb_newton_loop")

    out = {"device": torch.cuda.get_device_name(0), "power_limit": power_limit(),
           "workload": f"bench.py view {a.view}: 1920x1080, scale 2, no shading", "steps": []}
    print(f"{'step':>4} {'rows':>7} {'blocks':>8} {'iters':>5} {'kernel us/it':>12} "
          f"{'call us/it':>10}")
    for k, ((rows, blocks, iters, wall), ev) in enumerate(zip(steps, kernels)):
        kus = ev.time_range.elapsed_us()
        row = {"rows": rows, "blocks": blocks, "iterations": iters,
               "kernel_us": kus, "kernel_us_per_iter": kus / max(iters, 1),
               "call_us_per_iter": 1e6 * wall / max(iters, 1)}
        out["steps"].append(row)
        print(f"{k:>4} {rows:>7} {blocks:>8} {iters:>5} {row['kernel_us_per_iter']:>12.2f} "
              f"{row['call_us_per_iter']:>10.2f}")
    out["kernel_ms_total"] = sum(s["kernel_us"] for s in out["steps"]) / 1e3
    out["cg_iterations"] = sum(s["iterations"] for s in out["steps"])
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
