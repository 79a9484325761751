"""Time the fisheye and rational lens models of l3d_undistort_u8 on device-resident 3072 x 2304 images, and the existing pinhole cases
with this library and an earlier build of it, alternated in one process.

    python tools/bench_undistort_lens.py [--batches 26,200] [--reps 5] [--parent-lib PATH] [--rounds 3] [--out FILE]

Per image: CUDA events around `reps` launches on the context's stream after `warmup` launches, with the algorithmic traffic (C*W*H
bytes read + written) over the 3.35 TB/s data-sheet HBM3 figure and a lower bound on FP64 issue: the explicit IEEE adds and
multiplies per pixel of ud_fisheye_point / ud_map_point (sqrt, atan and the division are not counted) over 34 TFLOP/s, doubled
because nothing is contracted to a fused multiply-add.  --parent-lib: a libl3d_b200.so built from an earlier commit, whose
l3d_undistort_desc ends at tangential[2]; the two libraries time the bench_undistort.py pinhole cameras in alternation, `rounds` times.
The card name, power limit and max SM clock are read in the same run.
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_undistort import FP64_FLOPS, HBM_BPS, H, W, gpu_info  # noqa: E402

K = np.array([[1100.0, 0, 1536.0], [0, 1100.0, 1152.0], [0, 0, 1]])
# name: (make_undistort_desc keywords, explicit FP64 adds / multiplies per pixel)
LENSES = {
    "fisheye": (dict(model=1, fisheye=(0.05, -0.01, 0.003, -0.0005)), 22 + 1 / 16),
    "rational": (dict(radial=(0.12, -0.05, 0.01), tangential=(0.0007, -0.0004), rational=(0.08, -0.02, 0.005)), 36 + 3 / 16 + 3 / 128),
}
PINHOLE = {"k1": dict(radial=(-0.08, 0, 0)), "full": dict(radial=(0.1, -0.05, 0.02), tangential=(0.0012, -0.0021))}
K_PIN = np.array([[2800.0, 0, 1536.0], [0, 2800.0, 1152.0], [0, 0, 1]])


class ParentDesc(C.Structure):
    """l3d_undistort_desc before the lens fields"""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("channels", C.c_int32), ("src_pitch", C.c_int64), ("dst_pitch", C.c_int64),
                ("src", C.c_void_p), ("dst", C.c_void_p), ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("radial", C.c_double * 3), ("tangential", C.c_double * 2)]


class Lib:
    """one library's context: create, undistort on device, stream"""
    def __init__(self, path, desc_type):
        from line3dpp_b200 import capi
        self.L = capi.bind(C.CDLL(path), capi.HEADERS[:1])      # include/l3d_capi.h: the ABI both builds export
        self.h = C.c_void_p()
        assert self.L.l3d_ctx_create(0, C.byref(self.h)) == 0, path
        self.desc_type = desc_type

    def descs(self, src, dst, channels, K, kw):
        from line3dpp_b200 import capi
        n = src.shape[0]
        out = (self.desc_type * n)()
        row = W * channels
        for i in range(n):
            d = capi.make_undistort_desc(W, H, channels, K, src=src[i].data_ptr(), src_pitch=row, dst=dst[i].data_ptr(), dst_pitch=row, **kw)
            C.memmove(C.byref(out, i * C.sizeof(self.desc_type)), C.byref(d), C.sizeof(self.desc_type))
        return out

    def time(self, descs, reps, warmup):
        import torch
        stream = torch.cuda.ExternalStream(self.L.l3d_stream(self.h) or 0)
        for _ in range(warmup):
            assert self.L.l3d_undistort_u8(self.h, len(descs), descs, 1) == 0
        self.L.l3d_sync(self.h)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(reps):
            self.L.l3d_undistort_u8(self.h, len(descs), descs, 1)
        e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1) * 1e3 / (reps * len(descs))

    def close(self):
        self.L.l3d_ctx_destroy(self.h)


def images(channels, batch):
    import torch
    g = torch.Generator(device="cuda").manual_seed(channels * 1000 + batch)
    src = torch.randint(0, 256, (batch, H, W * channels), dtype=torch.uint8, device="cuda", generator=g)
    return src, torch.empty_like(src)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="26,200")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_undistort_lens: no CUDA device (nothing is timed on the CPU)")
    from line3dpp_b200 import capi
    new = Lib(capi._build.build(), capi.UndistortDesc)
    res = {"gpu": gpu_info(), "image": f"{W}x{H}", "lenses": [], "pinhole": []}
    batches = [int(b) for b in a.batches.split(",")]
    px = W * H
    for channels in (1, 3):
        for batch in batches:
            src, dst = images(channels, batch)
            for name, (kw, ops) in LENSES.items():
                us = new.time(new.descs(src, dst, channels, K if name == "fisheye" else K_PIN, kw), a.reps, a.warmup)
                t_hbm, t_fp64 = 2 * channels * px / HBM_BPS * 1e6, 2 * ops * px / FP64_FLOPS * 1e6
                r = {"lens": name, "channels": channels, "batch": batch, "us_per_image": round(us, 2), "hbm_datasheet_us": round(t_hbm, 2),
                     "fp64_unfused_floor_us": round(t_fp64, 2), "achieved_gbs": round(2 * channels * px / us * 1e-3, 1)}
                print(json.dumps(r), flush=True)
                res["lenses"].append(r)
            del src, dst
            torch.cuda.empty_cache()
    if a.parent_lib:
        old = Lib(a.parent_lib, ParentDesc)
        for channels in (1, 3):
            for batch in batches:
                src, dst = images(channels, batch)
                for cam, kw in PINHOLE.items():
                    dn, do = new.descs(src, dst, channels, K_PIN, kw), old.descs(src, dst, channels, K_PIN, kw)
                    t = {"new": [], "parent": []}
                    for _ in range(a.rounds):
                        t["new"].append(round(new.time(dn, a.reps, a.warmup), 2))
                        t["parent"].append(round(old.time(do, a.reps, a.warmup), 2))
                    r = {"camera": cam, "channels": channels, "batch": batch, **t}
                    print(json.dumps(r), flush=True)
                    res["pinhole"].append(r)
                del src, dst
                torch.cuda.empty_cache()
        old.close()
    new.close()
    res["gpu_after"] = gpu_info()
    print(json.dumps({"gpu": res["gpu"], "gpu_after": res["gpu_after"]}))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
