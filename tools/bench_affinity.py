"""Time l3d_affinity_matrix (kept list, candidates, unused() fixpoint, local ids, emission) at the benchmark's size, with and without
collinearity links, and print a SHA-256 of every affinity output so that two builds can be compared byte for byte.

    python tools/bench_affinity.py [--reps 5] [--warmup 1] [--out FILE]
    L3D_LIB=/path/to/other/libl3d_b200.so python tools/bench_affinity.py ...      # the same for another build of the library

Two scenes of 1000 views x 3000 segments, ring +-5 neighbours (BASELINE.json configs[3]): the plain one with links off, and one with
collinear fragments (synth collinear=True) with links at 2 px.  Each is matched (kNN 10) and scored once; then every timed call is
preceded by l3d_find_collinear switching the links off and on again (resp. on and off), which drops the cached matrix, and timed with
a host clock around the call and the stream synchronisation.  After timing, the digests cover l3d_affinity_edges (gi, gj, w),
l3d_affinity_matrix (CLEdge list and local2global) and l3d_rdd_affinity (10 iterations).  The card name and power limit are read
in the same run.
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

VIEWS, SEGS, RING, KNN, EPI = 1000, 3000, 5, 10, 0.25
TWO_SIGA_SQR, MIN_AFFINITY, COLLIN_PX = 200.0, 0.5, 2.0


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "nvidia-smi failed"
    except (OSError, subprocess.SubprocessError, IndexError):
        return "nvidia-smi unavailable"


def sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def scored_context(sc):
    from line3dpp_b200 import capi, synth
    V = sc.num_views
    RtKinv, Cw = synth.camera_blocks(sc)
    k = [2.5 / sc.K[v][0, 0] for v in range(V)]          # spatial regulariser of 2.5 px (View::getSpecificSpatialReg)
    descs = capi.make_view_descs(sc.cam_ids, [sc.width] * V, [sc.height] * V, [len(s) for s in sc.segs], RtKinv, Cw, Cw, k, sc.median_depth)
    pairs = synth.view_pairs(sc.neighbors, sc.cam_ids)
    F = np.stack([synth.fundamental(sc.K[s], sc.R[s], sc.t[s], sc.K[t], sc.R[t], sc.t[t]).astype(np.float32).reshape(9) for s, t in pairs])
    ctx = capi.Context(0)
    ctx.set_views(descs, sc.segs)
    ctx.match_pairs(pairs, F, EPI, KNN)
    ctx._chk(ctx.L.l3d_score_sweep(ctx.h, C.c_float(TWO_SIGA_SQR), C.c_float(.5), C.c_float(.75), C.c_float(.1)), "l3d_score_sweep")
    return ctx, float(np.median(sc.median_depth))


def run_scene(name, sc, links, reps, warmup):
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    ctx, med = scored_context(sc)
    L = ctx.L
    args = (ctx.h, C.c_float(TWO_SIGA_SQR), C.c_float(med), C.c_float(MIN_AFFINITY))
    nids = C.c_longlong(0)
    on, off = (COLLIN_PX, 0.0) if links else (0.0, COLLIN_PX)
    ms = []
    for r in range(warmup + reps):
        ctx.find_collinear(off, 0)
        ctx.find_collinear(on, 0)                        # a change of the links drops the cached matrix
        ctx.sync()
        t0 = time.perf_counter()
        n = ctx._chk(L.l3d_affinity_matrix(*args, None, None, None, C.c_longlong(0), None, C.c_longlong(0), C.byref(nids)), "l3d_affinity_matrix")
        ctx.sync()
        if r >= warmup:
            ms.append((time.perf_counter() - t0) * 1e3)
    ei, ej, ew, l2g = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.float32), np.zeros(nids.value, np.int64)
    ctx._chk(L.l3d_affinity_matrix(*args, p(ei), p(ej), p(ew), C.c_longlong(n), p(l2g), C.c_longlong(len(l2g)), C.byref(nids)), "l3d_affinity_matrix")
    oi, oj, ow = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.float32)
    ctx._chk(L.l3d_rdd_affinity(ctx.h, 10, p(oi), p(oj), p(ow), C.c_longlong(n)), "l3d_rdd_affinity")
    ne = ctx._chk(L.l3d_affinity_edges(*args, None, None, None, C.c_longlong(0)), "l3d_affinity_edges")
    gi, gj, w = np.zeros(ne, np.int64), np.zeros(ne, np.int64), np.zeros(ne, np.float32)
    ctx._chk(L.l3d_affinity_edges(*args, p(gi), p(gj), p(w), C.c_longlong(ne)), "l3d_affinity_edges")
    ctx.close()
    return dict(scene=name, links_px=COLLIN_PX if links else None, candidates=int(ne), matrix_entries=int(n), ids=int(nids.value),
                ms=[round(x, 3) for x in ms], median_ms=round(float(np.median(ms)), 3),
                sha256=dict(edges=sha(gi, gj, w), matrix=sha(ei, ej, ew, l2g), rdd=sha(oi, oj, ow)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from line3dpp_b200 import synth
    rows = [run_scene("plain", synth.make_scene(VIEWS, SEGS, 1004, f"ring{RING}"), False, a.reps, a.warmup),
            run_scene("collinear", synth.make_scene(VIEWS, SEGS, 1005, f"ring{RING}", collinear=True), True, a.reps, a.warmup)]
    res = dict(gpu=gpu_info(), lib=os.environ.get("L3D_LIB") or "in-tree", reps=a.reps, scenes=rows)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
