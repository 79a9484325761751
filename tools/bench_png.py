"""Batched PNG decoding of 3072 x 2304 photos on the GPU: per-kernel device time, readImagesGray end to end, and cv2 on the host.

    python tools/bench_png.py [--batches 1,8,32,128] [--reps 3] [--out DIR]

Inputs are built at run time from the two reference photos of tests/golden (jpeg_photo_*.jpg): each as a grey and as an RGB PNG,
written by cv2 at compression levels 1 and 6 (eight files, used round-robin).  Prints one JSON object: the GPU's name, power limit
and SM clock sampled during the run; the device time of k_png_inflate / k_png_unfilter / k_png_gray per photo from torch.profiler;
readImagesGray's wall time per photo at each batch size (median of --reps); and cv2.imread on the host's threads.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import threading
import time
from concurrent.futures import ThreadPoolExecutor

import cv2
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def smi(q):
    return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()[0]


class ClockSampler(threading.Thread):
    def __init__(self):
        super().__init__(daemon=True)
        self.samples, self.stop = [], threading.Event()

    def run(self):
        while not self.stop.is_set():
            try:
                self.samples.append(int(smi("clocks.sm").split()[0]))
            except (ValueError, IndexError):
                pass
            self.stop.wait(0.5)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="1,8,32,128")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from line3dpp_b200 import capi, line3d
    if not torch.cuda.is_available():
        raise SystemExit("bench_png needs a CUDA GPU")
    tmp = tempfile.mkdtemp()
    paths = []
    for k in range(2):
        bgr = cv2.imread(os.path.join(ROOT, "tests", "golden", f"jpeg_photo_{k}.jpg"), cv2.IMREAD_COLOR)
        for kind, img in (("grey", cv2.cvtColor(bgr, cv2.COLOR_BGR2GRAY)), ("rgb", bgr)):
            for lv in (1, 6):
                p = os.path.join(tmp, f"photo{k}_{kind}_l{lv}.png")
                cv2.imwrite(p, img, [cv2.IMWRITE_PNG_COMPRESSION, lv])
                paths.append(p)
    data = [open(p, "rb").read() for p in paths]
    # every input once: the GPU against cv2
    ref = [cv2.imread(p, cv2.IMREAD_GRAYSCALE) for p in paths]
    got = line3d.read_png_gray(paths)
    assert all(np.array_equal(g, r) for g, r in zip(got, ref)), "GPU output differs from cv2"
    sampler = ClockSampler()
    sampler.start()
    res = {"gpu": smi("name"), "power_limit": smi("power.limit"), "inputs": [os.path.basename(p) + f" ({len(d)} bytes)" for p, d in zip(paths, data)]}
    # device time per kernel: one context, a batch of 32
    ctx = capi.Context(0)
    batch = [data[i % len(data)] for i in range(32)]
    ctx.decode_png_gray(batch)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            ctx.decode_png_gray(batch)
    kern = {}
    for e in prof.key_averages():
        if e.key.startswith("k_png") or "k_png" in e.key:
            name = [n for n in ("k_png_inflate", "k_png_unfilter", "k_png_gray") if n in e.key][0]
            kern[name] = round(e.device_time_total / 1000.0 / (3 * 32), 3)
    res["kernel_ms_per_photo_batch32"] = kern
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        ctx.decode_png_gray([data[0]])
    res["kernel_ms_one_photo_" + os.path.basename(paths[0])] = {[n for n in ("k_png_inflate", "k_png_unfilter", "k_png_gray") if n in e.key][0]:
                                                              round(e.device_time_total / 1000.0, 3) for e in prof.key_averages() if "k_png" in e.key}
    ctx.close()
    # readImagesGray end to end (signature check, then one PNG batch)
    e2e = {}
    for b in [int(x) for x in a.batches.split(",")]:
        ps = [paths[i % len(paths)] for i in range(b)]
        line3d.read_image_gray(ps)
        ts = []
        for _ in range(a.reps):
            t = time.perf_counter()
            line3d.read_image_gray(ps)
            ts.append(time.perf_counter() - t)
        e2e[b] = round(1000 * float(np.median(ts)) / b, 2)
    res["readImagesGray_ms_per_photo"] = e2e
    # cv2 on the host: one thread on one photo, and all threads on 128
    t = time.perf_counter()
    for p in paths:
        cv2.imread(p, cv2.IMREAD_GRAYSCALE)
    res["cv2_one_thread_ms_per_photo"] = round(1000 * (time.perf_counter() - t) / len(paths), 2)
    nt = os.cpu_count()
    ps = [paths[i % len(paths)] for i in range(128)]
    with ThreadPoolExecutor(nt) as ex:
        t = time.perf_counter()
        list(ex.map(lambda p: cv2.imread(p, cv2.IMREAD_GRAYSCALE), ps))
        res[f"cv2_{nt}_threads_ms_per_photo_128"] = round(1000 * (time.perf_counter() - t) / 128, 2)
    sampler.stop.set()
    sampler.join()
    res["sm_clock_mhz"] = [min(sampler.samples), int(np.median(sampler.samples)), max(sampler.samples)] if sampler.samples else None
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_png.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
