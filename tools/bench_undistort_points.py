"""Time the lens undistortion of points (l3d_undistort_points, k_undistort_points) on device-resident float32 points, and addImage with
a lens against the three-call frontend loop it replaces.

    python tools/bench_undistort_points.py [--sizes 1e5,1e6,1e7,3e7] [--reps 5] [--views 26] [--out FILE]

Points: for every size and lens (radtan, 5 coefficients: five fixed iterations; fisheye: up to ten Newton steps and a tan), uniform over
a 3072 x 2304 image and 10% beyond it, one set per call.  Warm-up launches, then CUDA events around `reps` launches on the context's stream.
Reported per million points: the device time, the HBM floor (8 bytes read + 8 written per point over the 3.35 TB/s data-sheet HBM3
figure) and the FP64 issue floor (the double-precision instructions per point counted from the kernel source, a division counted as ten
and tan as forty, over 132 SMs x 64 FP64 lanes x the card's maximum SM clock).  Which floor is larger says what bounds the kernel.

addImage: `views` views of the 3072 x 2304 photos under tests/golden (cycled), each decoded on the GPU (read_image_gray), then either
undistort_image + add_image_pixels (the loop of INTEGRATION.md before this feature: a context per undistortImage call, the image to the
host and back) or add_image_pixels(..., lens=) (undistortion and preparation chained on the Line3D's context).  The detector returns a
fixed list, so neither path times a line detector; the segment cache is off.  Host wall-clock per view, after one warm-up view.
The card name, power limit and maximum SM clock are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

W, H = 3072, 2304
HBM_BPS = 3.35e12
SMS, FP64_LANES = 132, 64
DIV, TAN = 10, 40
# FP64 instructions per point from csrc/l3d_undistort.cu: radtan = prologue (normalise, tilt) + 5 x (r2, icdist, dx, dy, update) + the
# rectification; fisheye = prologue (two divisions, sqrt) + per Newton step (powers, numerator, denominator, division, update) + tan
RADTAN_OPS = 16 + 5 * (3 + 12 + DIV + 13 + 13 + 4) + 10 + DIV
FISHEYE_STEP_OPS = 4 + 4 + 6 + 8 + DIV + 2
FISHEYE_FIXED_OPS = 2 * DIV + 5 + DIV + 12 + 3 * DIV + TAN
LENSES = {"radtan": dict(model=0, k=(-0.12, 0.05, 0.0, 0, 0, 0), p=(0.001, -0.0007)),
          "fisheye": dict(model=1, k=(0.05, -0.01, 0.003, -0.0005), p=(0, 0))}
K = np.array([[2400.0, 0, 1530.5], [0, 2410.0, 1160.25], [0, 0, 1]])
FK = np.array([[1100.0, 0, 1536.0], [0, 1100.0, 1152.0], [0, 0, 1]])


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "nvidia-smi failed"
    except (OSError, subprocess.SubprocessError, IndexError):
        return "nvidia-smi unavailable"


def max_clock_hz(info):
    try:
        return float(info.split(",")[2].split()[0]) * 1e6
    except (IndexError, ValueError):
        return 1.98e9


def newton_steps(pts, Kc, lens):
    """mean Newton steps per fisheye point (from the numpy restatement, on a sample)"""
    sample = pts[:: max(1, len(pts) // 20000)]
    k = list(lens["k"])[:4]
    u = sample[:, 0].astype(np.float64)
    v = sample[:, 1].astype(np.float64)
    pwx, pwy = (u - Kc[0, 2]) / Kc[0, 0], (v - Kc[1, 2]) / Kc[1, 1]
    td = np.minimum(np.sqrt(pwx * pwx + pwy * pwy), np.pi / 2)
    theta, steps, live = td.copy(), np.zeros(len(td)), td > 1e-8
    for _ in range(10):
        t2 = theta * theta
        a, b, c, d = k[0] * t2, k[1] * t2 ** 2, k[2] * t2 ** 3, k[3] * t2 ** 4
        fix = (theta * (1 + a + b + c + d) - td) / (1 + 3 * a + 5 * b + 7 * c + 9 * d)
        theta = np.where(live, theta - fix, theta)
        steps += live
        live &= ~(np.abs(fix) < 1e-8)
    return float(steps.mean())


def time_points(ctx, n, lens_name, reps, warmup, clock):
    import torch
    from line3dpp_b200 import capi
    lens = LENSES[lens_name]
    Kc = K if lens_name == "radtan" else FK
    g = torch.Generator(device="cuda").manual_seed(n % 1000003)
    src = torch.rand((n, 2), generator=g, device="cuda", dtype=torch.float32)
    src[:, 0] = src[:, 0] * (1.2 * W) - 0.1 * W
    src[:, 1] = src[:, 1] * (1.2 * H) - 0.1 * H
    dst = torch.empty_like(src)
    torch.cuda.synchronize()
    descs = (capi.PointsDesc * 1)(capi.make_points_desc(Kc, lens, n, src.data_ptr(), dst.data_ptr()))
    stream = torch.cuda.ExternalStream(ctx.stream)
    for _ in range(warmup):
        ctx.undistort_points_descs(descs, 1)
    ctx.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(reps):
        ctx.undistort_points_descs(descs, 1)
    e1.record(stream)
    e1.synchronize()
    us_per_m = e0.elapsed_time(e1) * 1e3 / reps / (n / 1e6)
    if lens_name == "radtan":
        ops = RADTAN_OPS
    else:
        ops = FISHEYE_FIXED_OPS + newton_steps(src[: min(n, 200000)].cpu().numpy(), Kc, lens) * FISHEYE_STEP_OPS
    hbm_us = 16 * 1e6 / HBM_BPS * 1e6
    fp64_us = ops * 1e6 / (SMS * FP64_LANES * clock) * 1e6
    return {"lens": lens_name, "points": n, "us_per_million": round(us_per_m, 2), "hbm_floor_us_per_million": round(hbm_us, 2),
            "fp64_issue_floor_us_per_million": round(fp64_us, 2), "fp64_ops_per_point": round(ops, 1),
            "share_of_larger_floor": round(max(hbm_us, fp64_us) / us_per_m, 3)}


def time_add_image(views):
    from line3dpp_b200 import line3d
    photos = [os.path.join(ROOT, "tests", "golden", f"jpeg_photo_{i}.jpg") for i in (0, 1)]
    lens = LENSES["radtan"]
    det = np.array([[10, 10, 900, 700], [50, 1200, 2000, 1300], [3000, 100, 2500, 2200]], np.float32)
    out = {}
    for mode in ("three_calls", "lens"):
        with tempfile.TemporaryDirectory() as tmp:
            L = line3d.Line3D(True, True, output_folder=tmp, load_segments=False)
            L.set_segment_detector(lambda g: det * np.float32(g.shape[1] / W))
            times = []
            for v in range(views + 1):
                t0 = time.perf_counter()
                img = line3d.read_image_gray(photos[v % 2])
                if mode == "three_calls":
                    L.add_image_pixels(v, line3d.undistort_image(img, K, lens), K, np.eye(3), np.array([0, 0, 1.0]), 2.0, [1])
                else:
                    L.add_image_pixels(v, img, K, np.eye(3), np.array([0, 0, 1.0]), 2.0, [1], lens=lens)
                times.append(time.perf_counter() - t0)
            L.close()
        out[mode] = {"ms_per_view": round(1e3 * float(np.mean(times[1:])), 2), "views": views}
    out["speedup"] = round(out["three_calls"]["ms_per_view"] / out["lens"]["ms_per_view"], 2)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1e5,1e6,1e7,3e7")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--views", type=int, default=26)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from line3dpp_b200 import capi
    info = gpu_info()
    clock = max_clock_hz(info)
    ctx = capi.Context(0)
    res = {"gpu": info, "points": [], "add_image": None}
    for lens_name in LENSES:
        for n in (int(float(s)) for s in a.sizes.split(",")):
            r = time_points(ctx, n, lens_name, a.reps, a.warmup, clock)
            print(json.dumps(r), flush=True)
            res["points"].append(r)
    ctx.close()
    res["add_image"] = time_add_image(a.views)
    print(json.dumps(res["add_image"]), flush=True)
    print("gpu:", info)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
