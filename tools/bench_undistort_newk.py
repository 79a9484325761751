"""Time l3d_undistort_u8 into a new camera matrix and size: device-resident 3072 x 2304 fisheye and radtan images into several output
sizes, with the new K from the host new-camera-matrix functions, and the zero-tail calls of all three lens kinds against an earlier build
of this library, alternated in one process.

    python tools/bench_undistort_newk.py [--batch 26] [--reps 5] [--parent-lib PATH] [--rounds 3] [--out FILE]

Per image: CUDA events around `reps` launches on the context's stream after `warmup` launches.  The floor is the algorithmic traffic
over the 3.35 TB/s data-sheet HBM3 figure: each output pixel written once, and every source pixel the map reaches read once (counted
from the map itself, so a smaller output that reaches less of the source has a lower floor).  --parent-lib: a libl3d_b200.so built from
an earlier commit, whose l3d_undistort_desc ends at fisheye[4].  The card name, power limit and max SM clock are read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_undistort import HBM_BPS, H, W, gpu_info  # noqa: E402
from tools.bench_undistort_lens import Lib, images  # noqa: E402

K_FE = np.array([[800.0, 0, 1536.0], [0, 800.0, 1152.0], [0, 0, 1]])
FE = {"model": 1, "k": [0.05, -0.01, 0.002, -0.0005, 0, 0], "p": [0, 0]}
K_RT = np.array([[2500.0, 0, 1536.0], [0, 2500.0, 1152.0], [0, 0, 1]])
RT = {"model": 0, "k": [-0.2, 0.05, 0.01, 0, 0, 0], "p": [0.001, -0.0007]}
RA = {"model": 0, "k": [0.12, -0.05, 0.01, 0.08, -0.02, 0.005], "p": [0.0007, -0.0004]}
OUT_SIZES = [(1536, 1152), (3072, 2304), (4096, 3072), (4000, 1500)]


def new_k(name, out_size):
    from line3dpp_b200 import line3d
    if name == "fisheye":
        return line3d.fisheye_new_camera_matrix(K_FE, FE, (W, H), 0.0, out_size)
    return line3d.optimal_new_camera_matrix(K_RT, RT, (W, H), 1.0, out_size)[0]


def descs(lib, src, dst, channels, K, lens, nk, out_size):
    """lib's descriptors for the batch; the new-K fields only where lib's descriptor has them"""
    from line3dpp_b200 import capi
    n, ow, oh = src.shape[0], out_size[0], out_size[1]
    out = (lib.desc_type * n)()
    for i in range(n):
        d = capi.make_undistort_desc(W, H, channels, K, src=src[i].data_ptr(), src_pitch=W * channels, dst=dst[i].data_ptr(), dst_pitch=ow * channels,
                                     new_K=nk, out_size=None if nk is None else out_size, **capi.lens_desc_args(lens))
        C.memmove(C.byref(out, i * C.sizeof(lib.desc_type)), C.byref(d), C.sizeof(lib.desc_type))
    return out


def source_reached(ctx, K, lens, nk, out_size, channels):
    """bytes of the source the map reaches (each source pixel under any of an output pixel's four taps, counted once)"""
    xy, fr = ctx.undistort_map(W, H, K, lens=lens, new_K=nk, out_size=out_size)
    x, y = xy[..., 0].astype(np.int64), xy[..., 1].astype(np.int64)
    hit = np.zeros((H + 1, W + 1), bool)
    for dx in (0, 1):
        for dy in (0, 1):
            ok = (x + dx >= 0) & (x + dx < W) & (y + dy >= 0) & (y + dy < H)
            hit[(y + dy)[ok], (x + dx)[ok]] = True
    return int(hit.sum()) * channels


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=26)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_undistort_newk: no CUDA device (nothing is timed on the CPU)")
    from line3dpp_b200 import capi
    new = Lib(capi._build.build(), capi.UndistortDesc)
    ctx = capi.Context(0)
    res = {"gpu": gpu_info(), "image": f"{W}x{H}", "batch": a.batch, "new_k": [], "zero_tail": []}
    for channels in (1, 3):
        src, _ = images(channels, a.batch)
        for name, K, lens in (("fisheye", K_FE, FE), ("radtan", K_RT, RT)):
            for out_size in OUT_SIZES:
                nk = new_k(name, out_size)
                dst = torch.empty((a.batch, out_size[1], out_size[0] * channels), dtype=torch.uint8, device="cuda")
                us = new.time(descs(new, src, dst, channels, K, lens, nk, out_size), a.reps, a.warmup)
                nbytes = source_reached(ctx, K, lens, nk, out_size, channels) + out_size[0] * out_size[1] * channels
                r = {"lens": name, "channels": channels, "out": f"{out_size[0]}x{out_size[1]}", "f_new": round(float(nk[0, 0]), 2),
                     "us_per_image": round(us, 2), "hbm_datasheet_us": round(nbytes / HBM_BPS * 1e6, 2), "achieved_gbs": round(nbytes / us * 1e-3, 1)}
                print(json.dumps(r), flush=True)
                res["new_k"].append(r)
                del dst
        del src
        torch.cuda.empty_cache()
    if a.parent_lib:
        parent_desc = type("ParentDesc", (C.Structure,), {"_fields_": capi.UndistortDesc._fields_[:-6]})
        old = Lib(a.parent_lib, parent_desc)
        for channels in (1, 3):
            src, dst = images(channels, a.batch)
            for name, K, lens in (("fisheye", K_FE, FE), ("radtan", K_RT, RT), ("rational", K_RT, RA)):
                dn, do = descs(new, src, dst, channels, K, lens, None, (W, H)), descs(old, src, dst, channels, K, lens, None, (W, H))
                t = {"new": [], "parent": []}
                for _ in range(a.rounds):
                    t["new"].append(round(new.time(dn, a.reps, a.warmup), 2))
                    t["parent"].append(round(old.time(do, a.reps, a.warmup), 2))
                r = {"lens": name, "channels": channels, **t}
                print(json.dumps(r), flush=True)
                res["zero_tail"].append(r)
            del src, dst
            torch.cuda.empty_cache()
        old.close()
    ctx.close()
    new.close()
    res["gpu_after"] = gpu_info()
    print(json.dumps({"gpu": res["gpu"], "gpu_after": res["gpu_after"]}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
