"""Time the tie-point triangulation (l3d_triangulate_points, k_triangulate) on device-resident observations, next to the CPU restatement
(numpy: A^T A per point, batched eigh) on the host threads.

    python tools/bench_triangulate.py [--reps 20] [--cams 500] [--out FILE]

Two workloads: 10^6 points x 8 observations and 10^5 points x 40, observed by `cams` cameras on a ring (500: the matrices are staged in
shared memory).  GPU: warm-up launches, then CUDA events around `reps` launches on the context's stream.  Reported next to each time:
the HBM bytes the kernel must move (20 B per observation: camera id + xy; 36 B per point: CSR offset, X, flag; the camera matrices are
gathered from shared memory) over the 3.35 TB/s data-sheet HBM3 figure, and the double-precision operations of a model count
(56 per observation for the rows and the 10 products of A^T A, 1600 per point for four Jacobi sweeps and the division) over the
34 TFLOP/s data-sheet FP64 (non-tensor) figure.  That figure counts a fused multiply-add as two operations; the library is compiled
without contraction, so the issue floor of this code is twice the data-sheet time (`fp64_unfused_ms`).  The card name and power limit
are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BPS, FP64_FLOPS = 3.35e12, 34e12
FLOPS_PER_OBS, FLOPS_PER_POINT = 56, 1600
WORKLOADS = ((1000000, 8), (100000, 40))


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "nvidia-smi failed"
    except (OSError, subprocess.SubprocessError, IndexError):
        return "nvidia-smi unavailable"


def problem(n, k, ncam, seed):
    """n points in [-5, 5]^3, each seen by k distinct cameras of a ring of ncam (f = 1200 px), 0.5 px noise"""
    rng = np.random.default_rng(seed)
    K = np.array([[1200.0, 0, 960], [0, 1200.0, 540], [0, 0, 1]])
    ang = np.linspace(0, 2 * np.pi, ncam, endpoint=False)
    Cs = np.stack([30 * np.cos(ang), 30 * np.sin(ang), 10 + 2 * np.sin(3 * ang)], 1)
    P = []
    for C in Cs:
        z = -C / np.linalg.norm(C); x = np.cross([0.0, 0.0, 1.0], z); x /= np.linalg.norm(x)
        R = np.stack([x, np.cross(z, x), z])
        P.append(K @ np.hstack([R, (-R @ C)[:, None]]))
    P = np.stack(P)
    X = rng.uniform(-5, 5, (n, 3))
    cam = (rng.integers(0, ncam, (n, 1)) + np.arange(k)[None, :] * max(1, ncam // k)) % ncam
    cam = cam.reshape(-1).astype(np.int32)
    h = np.einsum("nij,nj->ni", P[cam], np.hstack([np.repeat(X, k, 0), np.ones((n * k, 1))]))
    xy = h[:, :2] / h[:, 2:] + rng.normal(0, 0.5, (n * k, 2))
    ptr = np.arange(n + 1, dtype=np.int64) * k
    return ptr, cam, xy, P


def cpu_restatement(ptr, cam, xy, P, threads):
    """A^T A of every point and its smallest eigenvector (numpy eigh), chunks on `threads` host threads"""
    n = len(ptr) - 1
    k = int(ptr[1] - ptr[0])

    def chunk(a, b):
        Pc = P[cam[a * k:b * k]]
        x = xy[a * k:b * k]
        r1 = -Pc[:, 1] + x[:, 1:2] * Pc[:, 2]; r2 = Pc[:, 0] - x[:, 0:1] * Pc[:, 2]
        A = (np.einsum("ni,nj->nij", r1, r1) + np.einsum("ni,nj->nij", r2, r2)).reshape(b - a, k, 4, 4).sum(1)
        v = np.linalg.eigh(A)[1][:, :, 0]
        return v[:, :3] / v[:, 3:]

    step = max(1, (n + threads * 4 - 1) // (threads * 4))
    with ThreadPoolExecutor(threads) as ex:
        return np.concatenate(list(ex.map(lambda a: chunk(a, min(n, a + step)), range(0, n, step))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cams", type=int, default=500)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from line3dpp_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("bench_triangulate: no CUDA device (the triangulation runs on the GPU only)")
    ctx = capi.Context(0)
    stream = torch.cuda.ExternalStream(ctx.stream)
    threads = os.cpu_count() or 1
    rows = []
    for n, k in WORKLOADS:
        ptr, cam, xy, P = problem(n, k, a.cams, seed=n + k)
        d = {name: torch.from_numpy(np.ascontiguousarray(v)).cuda() for name, v in (("ptr", ptr), ("cam", cam), ("xy", xy), ("P", P.reshape(-1, 12)))}
        X = torch.empty((n, 3), dtype=torch.float64, device="cuda")
        valid = torch.empty(n, dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        launch = lambda: ctx.triangulate_points_device(n, d["ptr"].data_ptr(), d["cam"].data_ptr(), d["xy"].data_ptr(), a.cams, d["P"].data_ptr(),
                                                       X.data_ptr(), valid.data_ptr())
        for _ in range(a.warmup):
            launch()
        ctx.sync()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(a.reps):
            launch()
        e1.record(stream)
        e1.synchronize()
        gpu_ms = e0.elapsed_time(e1) / a.reps
        t0 = time.perf_counter()
        Xc = cpu_restatement(ptr, cam, xy, P, threads)
        cpu_ms = (time.perf_counter() - t0) * 1e3
        Xg = X.cpu().numpy()
        rel = float(np.max(np.linalg.norm(Xg - Xc, axis=1) / np.linalg.norm(Xc, axis=1)))
        obs = n * k
        hbm_bytes = 20 * obs + 36 * n
        flops = FLOPS_PER_OBS * obs + FLOPS_PER_POINT * n
        rows.append(dict(points=n, obs_per_point=k, cameras=a.cams, gpu_ms=round(gpu_ms, 4), cpu_ms=round(cpu_ms, 1), cpu_threads=threads,
                         speedup=round(cpu_ms / gpu_ms, 1), max_rel_diff_vs_cpu=rel, hbm_bytes=hbm_bytes,
                         hbm_bound_ms=round(hbm_bytes / HBM_BPS * 1e3, 4), model_fp64_flops=flops, fp64_datasheet_ms=round(flops / FP64_FLOPS * 1e3, 4),
                         fp64_unfused_ms=round(2 * flops / FP64_FLOPS * 1e3, 4), valid=int(valid.sum().item())))
        print(json.dumps(rows[-1]), flush=True)
    res = dict(gpu=gpu_info(), reps=a.reps, workloads=rows)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))
    ctx.close()


if __name__ == "__main__":
    main()
