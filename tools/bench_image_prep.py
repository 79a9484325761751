"""Time the batched image preparation for line detection (l3d_prepare_gray_u8, k_prepare_gray_u8) on device-resident 3072 x 2304
images, the size of the reference's test images.

    python tools/bench_image_prep.py [--batches 26,200] [--reps 5] [--out FILE]

For grey and RGB images, max_img_width -1 (grey conversion / copy only) and 1920 (INTER_LINEAR to 1920 x 1440), and every batch size:
warm-up launches, then CUDA events around `reps` launches on the context's stream.  Per image it reports the time and the HBM floor:
the algorithmic traffic (C*W*H bytes read once + the prepared image written once) over the 3.35 TB/s data-sheet HBM3 figure.  The
card name, power limit and maximum SM clock are read in the same run.  When cv2 is importable, the reference's CPU path (cvtColor +
resize, one image) is timed for scale.
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
HBM_BPS = 3.35e12
MAX_WIDTHS = (-1, 1920)


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "nvidia-smi failed"
    except (OSError, subprocess.SubprocessError, IndexError):
        return "nvidia-smi unavailable"


def time_gpu(ctx, channels, batch, mw, reps, warmup):
    import torch
    from line3dpp_b200 import capi
    ow, oh, _ = capi.image_prep_size(W, H, mw)
    g = torch.Generator(device="cuda").manual_seed(channels * 1000 + batch)
    src = torch.randint(0, 256, (batch, H, W * channels), dtype=torch.uint8, device="cuda", generator=g)
    dst = torch.empty((batch, oh, ow), dtype=torch.uint8, device="cuda")
    descs = (capi.ImagePrepDesc * batch)()
    for i in range(batch):
        descs[i] = capi.make_image_prep_desc(W, H, channels, mw, src[i].data_ptr(), W * channels, dst[i].data_ptr(), ow)
    stream = torch.cuda.ExternalStream(ctx.stream)
    for _ in range(warmup):
        ctx.prepare_gray_device(descs)
    ctx.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(reps):
        ctx.prepare_gray_device(descs)
    e1.record(stream)
    e1.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / (reps * batch)
    nbytes = channels * W * H + ow * oh
    t_hbm = nbytes / HBM_BPS * 1e6
    return {"channels": channels, "batch": batch, "max_img_width": mw, "out": f"{ow}x{oh}", "us_per_image": round(us, 2),
            "hbm_bytes": nbytes, "hbm_floor_us": round(t_hbm, 2), "achieved_gbs": round(nbytes / us * 1e-3, 1),
            "frac_of_hbm_floor": round(t_hbm / us, 3)}


def time_cv2(channels, mw, reps=3):
    import cv2
    img = np.random.default_rng(channels).integers(0, 256, (H, W, channels) if channels == 3 else (H, W), dtype=np.uint8)
    best = None
    for _ in range(reps):
        t = time.perf_counter()
        g = cv2.cvtColor(img, cv2.COLOR_RGB2GRAY) if channels == 3 else img.copy()
        if mw > 0 and max(W, H) > mw:
            s = np.float32(mw) / np.float32(max(W, H))
            cv2.resize(g, None, fx=float(s), fy=float(s))
        dt = (time.perf_counter() - t) * 1e3
        best = dt if best is None else min(best, dt)
    return {"channels": channels, "max_img_width": mw, "ms_per_image": round(best, 3), "threads": cv2.getNumThreads(), "cv2": cv2.__version__}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="26,200")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_image_prep: no CUDA device (nothing is timed on the CPU)")
    from line3dpp_b200 import capi
    ctx = capi.Context(0)
    res = {"gpu": gpu_info(), "image": f"{W}x{H}", "rows": []}
    for channels in (1, 3):
        for batch in [int(b) for b in a.batches.split(",")]:
            for mw in MAX_WIDTHS:
                r = time_gpu(ctx, channels, batch, mw, a.reps, a.warmup)
                print(json.dumps(r), flush=True)
                res["rows"].append(r)
                torch.cuda.empty_cache()
    try:
        import cv2  # noqa: F401
        res["cv2_cpu"] = [time_cv2(c, mw) for c in (1, 3) for mw in MAX_WIDTHS]
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
