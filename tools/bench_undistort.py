"""Time the batched lens undistortion (l3d_undistort_u8, k_undistort_u8) on device-resident 3072 x 2304 images, the size of the
reference's test images.

    python tools/bench_undistort.py [--batches 26,200] [--reps 5] [--out FILE]

For grey and RGB images, a VisualSfM-style camera (k1 only) and a full five-coefficient one, and every batch size: warm-up launches,
then CUDA events around `reps` launches on the context's stream.  Per image it reports the time, the algorithmic traffic (C*W*H bytes
read + C*W*H written) over the 3.35 TB/s data-sheet HBM3 figure, and the double-precision operations per pixel counted from
ud_map_point (l3d_undistort.cu) over the 34 TFLOP/s data-sheet FP64 (non-tensor) figure.  That figure counts a fused multiply-add as
two operations; this code is compiled without contraction, so every add or multiply takes a whole FP64 issue slot and the issue floor
is twice the data-sheet time (`fp64_unfused_us`).  The card name and power limit are read in the same run.  When cv2 is importable,
the reference's CPU path (initUndistortRectifyMap + remap, one image) is timed as well.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

W, H = 3072, 2304
HBM_BPS, FP64_FLOPS = 3.35e12, 34e12
K = np.array([[2800.0, 0, 1536.0], [0, 2800.0, 1152.0], [0, 0, 1]])
# (radial, tangential, double operations per pixel in ud_map_point: r2, kr, xd, yd, u, v and the two *32 of ud_fix; the per-column
# x, x*x and per-row y, y*y are shared by a tile's 16 rows / 128 columns and add 3/16 + 3/128)
CAMERAS = {"k1": ((-0.08, 0, 0), (0, 0), 11 + 3 / 16 + 3 / 128),
           "full": ((0.1, -0.05, 0.02), (0.0012, -0.0021), 29 + 3 / 16 + 3 / 128)}


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "nvidia-smi failed"
    except (OSError, subprocess.SubprocessError, IndexError):
        return "nvidia-smi unavailable"


def time_gpu(ctx, channels, batch, cam, reps, warmup):
    import torch
    radial, tangential, ops = CAMERAS[cam]
    g = torch.Generator(device="cuda").manual_seed(channels * 1000 + batch)
    src = torch.randint(0, 256, (batch, H, W * channels), dtype=torch.uint8, device="cuda", generator=g)
    dst = torch.empty_like(src)
    from line3dpp_b200 import capi
    descs = (capi.UndistortDesc * batch)()
    row = W * channels
    for i in range(batch):
        descs[i] = capi.make_undistort_desc(W, H, channels, K, radial, tangential, src[i].data_ptr(), row, dst[i].data_ptr(), row)
    stream = torch.cuda.ExternalStream(ctx.stream)
    for _ in range(warmup):
        ctx.undistort_device(descs)
    ctx.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(reps):
        ctx.undistort_device(descs)
    e1.record(stream)
    e1.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / (reps * batch)
    px = W * H
    t_hbm = 2 * channels * px / HBM_BPS * 1e6
    t_fp64 = ops * px / FP64_FLOPS * 1e6
    return {"channels": channels, "batch": batch, "camera": cam, "us_per_image": round(us, 2),
            "hbm_bytes": 2 * channels * px, "hbm_datasheet_us": round(t_hbm, 2), "achieved_gbs": round(2 * channels * px / us * 1e-3, 1),
            "fp64_ops_per_px": round(ops, 2), "fp64_datasheet_us": round(t_fp64, 2), "fp64_unfused_us": round(2 * t_fp64, 2),
            "bound": "fp64" if 2 * t_fp64 > t_hbm else "hbm", "frac_of_bound": round(max(2 * t_fp64, t_hbm) / us, 3)}


def time_cv2(channels, reps=3):
    import cv2
    img = np.random.default_rng(channels).integers(0, 256, (H, W, channels) if channels == 3 else (H, W), dtype=np.uint8)
    dist = np.array([-0.08, 0, 0, 0, 0.0])
    best = None
    for _ in range(reps):
        t = time.perf_counter()
        m1, m2 = cv2.initUndistortRectifyMap(K, dist, np.eye(3), K, (W, H), cv2.CV_16SC2)
        cv2.remap(img, m1, m2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
        dt = (time.perf_counter() - t) * 1e3
        best = dt if best is None else min(best, dt)
    return {"channels": channels, "ms_per_image": round(best, 2), "threads": cv2.getNumThreads(), "cv2": cv2.__version__}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="26,200")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_undistort: no CUDA device (nothing is timed on the CPU)")
    from line3dpp_b200 import capi
    ctx = capi.Context(0)
    res = {"gpu": gpu_info(), "image": f"{W}x{H}", "rows": []}
    for channels in (1, 3):
        for batch in [int(b) for b in a.batches.split(",")]:
            for cam in CAMERAS:
                r = time_gpu(ctx, channels, batch, cam, a.reps, a.warmup)
                print(json.dumps(r), flush=True)
                res["rows"].append(r)
                torch.cuda.empty_cache()
    try:
        import cv2  # noqa: F401
        res["cv2_cpu"] = [time_cv2(1), time_cv2(3)]
    except ImportError:
        res["cv2_cpu"] = "cv2 absent on this host: the reference's CPU path was not timed"
    res["gpu_after"] = gpu_info()
    ctx.close()
    print(json.dumps({k: v for k, v in res.items() if k != "rows"}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
