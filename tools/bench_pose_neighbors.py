"""Time l3d_pose_neighbors: the device phases (per kernel, torch.profiler) and the host selection, on ring and grid-survey scenes of 1000
and 5000 views, and set the observation kernel against the FP64 issue bound of the H100 SXM data sheet.

    python tools/bench_pose_neighbors.py [--views 1000 5000] [--gx 32 --gy 24] [--reps 3] [--out FILE.json]

Observation work: the count and the fill pass each project every virtual point into every other view: 2 * V * (V - 1) * G
projections of 26 IEEE double adds and multiplies (R X + t: 18, K c: 8; -fmad=false, so no fused ops) and up to two divisions.  The
bound counts those 26 plus one per division as single FP64 issues: 132 SMs x 64 FP64 lanes x the SM clock (data sheet: 1.98 GHz boost,
33.5 TFLOP/s FP64 counting an FMA as two).  Needs a GPU; nothing falls back."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from line3dpp_b200 import capi  # noqa: E402
from tests import pose_model as pm  # noqa: E402

OPS_PER_PROJECTION = 28           # 18 + 8 adds / multiplies, 2 divisions counted once each
FP64_LANES = 132 * 64


def scene(kind, V):
    """ring: a closed loop of V forward-looking views 0.5 units apart (a vehicle or walk-through sequence), depth 5; grid: a nadir
    survey at height 40 with 10-unit spacing (about 80 % forward and 75 % side overlap)"""
    if kind == "ring":
        rad = 0.5 * V / (2.0 * np.pi)
        Rs, ts = [], []
        for i in range(V):
            th = 2.0 * np.pi * i / V
            C = np.array([rad * np.cos(th), 0.0, rad * np.sin(th)])
            R, t = pm.look_at(C, C + np.array([-np.sin(th), 0.0, np.cos(th)]))
            Rs.append(R); ts.append(t)
        return pm.Views(np.arange(V), np.repeat(pm.intrinsics(1000.0, 1920, 1080)[None], V, 0), Rs, ts, 1920, 1080, 5.0)
    nx = int(round(np.sqrt(V * 4 / 3)))
    return pm.grid_survey(nx, V // nx, spacing=10.0, height=40.0, w=4000, h=3000, f=3000.0, seed=2)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def kernel_times(ctx, d, gx, gy):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ctx.pose_neighbors(d, 10, gx, gy)
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            name = e.name.split("(")[0]
            out[name] = out.get(name, 0.0) + e.device_time_total / 1000.0
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, nargs="+", default=[1000, 5000])
    ap.add_argument("--gx", type=int, default=32)
    ap.add_argument("--gy", type=int, default=24)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    G = a.gx * a.gy
    info = gpu_info()
    print("GPU:", info)
    ctx = capi.Context(0)
    rows = []
    for kind in ("ring", "grid"):
        for V in a.views:
            Vs = scene(kind, V)
            V = len(Vs)
            d = capi.make_pose_views(Vs.cam_ids, Vs.K, Vs.R, Vs.t, Vs.width, Vs.height, Vs.depth)
            ctx.pose_neighbors(d, 10, a.gx, a.gy)                         # warm-up
            dev, host, wall = [], [], []
            for _ in range(a.reps):
                t0 = time.perf_counter()
                nb, n, (dms, hms) = ctx.pose_neighbors(d, 10, a.gx, a.gy)
                wall.append((time.perf_counter() - t0) * 1e3)
                dev.append(dms); host.append(hms)
            kt = kernel_times(ctx, d, a.gx, a.gy)
            obs_ms = sum(v for k, v in kt.items() if "k_pose_observe" in k)
            proj = 2.0 * V * (V - 1) * G
            bound_ms = proj * OPS_PER_PROJECTION / (FP64_LANES * 1.98e9) * 1e3     # at the data sheet's boost clock
            r = dict(scene=kind, views=V, G=G, device_ms=float(np.median(dev)), host_select_ms=float(np.median(host)),
                     call_ms=float(np.median(wall)), kernels_ms=kt, observe_ms=obs_ms, projections=proj, fp64_bound_ms=bound_ms, fp64_share=bound_ms / obs_ms if obs_ms else None,
                     mean_observers=float(n.sum()) / (V * G), mean_neighbors=float(np.mean([len(x) for x in nb])))
            print(json.dumps(r))
            rows.append(r)
    ctx.close()
    res = dict(gpu=info, ops_per_projection=OPS_PER_PROJECTION, fp64_lanes=FP64_LANES, rows=rows)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
