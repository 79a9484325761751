"""Time Line3D::matchImages on device lists against each other at the benchmark's size, and check that every list gives the same result.

    python tools/bench_multidevice.py --out DIR [--runs 3] [--devices 0 --devices 0,0 ...]

Workload: BASELINE.json configs[3]-shaped, 1000 views x 3000 segments, ring +-5 neighbours (synth seed 1003), kNN 10, through
L3DPP::Line3D.  Every --devices list is one arm (default: "0" and "0,0"); the arms alternate, `runs` times each.  A run constructs the
Line3D, adds the views, and calls matchImages; it reports the stats' ms_match (views upload, matching on every device, gather, host
clock), ms_score (scoring sweep) and ms_gather (CUDA events around l3d_match_gather on the primary's stream).  The first run of every
arm also reconstructs the 3D lines (no diffusion, no collinearity) and hashes the estimates, the kept matches of every view and the 3D
segments; the arms must agree byte for byte.  The card name, power limit and maximum SM clock are read in the same run (query only).
Writes DIR/multidevice.json and prints it.
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

VIEWS, SEGS, SEED, RING, KNN = 1000, 3000, 1003, 5, 10


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines() if r.returncode == 0 else ["nvidia-smi failed"]
    except (OSError, subprocess.SubprocessError):
        return ["nvidia-smi unavailable"]


def digest(L, scene):
    h = {k: hashlib.sha256() for k in ("estimates", "kept", "segments3d")}
    best, p = L.estimates()
    h["estimates"].update(best.tobytes()); h["estimates"].update(p.tobytes())
    for c in scene.cam_ids:
        h["kept"].update(L.view_matches(c, True).tobytes())
    h["segments3d"].update(L.segments3d().tobytes()); h["segments3d"].update(L.residuals().tobytes())
    return {k: v.hexdigest() for k, v in h.items()}


def run(scene, devices, check):
    from line3dpp_b200 import line3d
    L = line3d.Line3D(neighbors_by_worldpoints=False, devices=devices)
    try:
        L.add_scene(scene)
        L.match_images(knn=KNN)
        st = L.stats()
        out = {k: st[k] for k in ("ms_match", "ms_score", "ms_gather", "pair_evaluations", "matches_after_knn", "view_pairs")}
        if check:
            L.reconstruct_3d_lines(3, False, -1.0)
            out["lines3D"] = L.stats()["lines3D"]
            out["digest"] = digest(L, scene)
        return out
    finally:
        L.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--devices", action="append", help="comma-separated device list, one arm each (default: 0 and 0,0)")
    a = ap.parse_args()
    arms = [[int(x) for x in s.split(",")] for s in (a.devices or ["0", "0,0"])]
    from line3dpp_b200 import synth
    gpus = gpu_info()
    small = synth.make_scene(20, 300, 7, "ring3")
    for arm in arms:                                   # module loads and first-launch costs outside the timed runs
        run(small, arm, False)
    scene = synth.make_scene(VIEWS, SEGS, SEED, f"ring{RING}")
    res = {str(arm): [] for arm in arms}
    for r in range(a.runs):
        for arm in arms:
            res[str(arm)].append(run(scene, arm, r == 0))
            print(f"run {r} devices {arm}: " + json.dumps({k: v for k, v in res[str(arm)][-1].items() if k != "digest"}), flush=True)
    digests = [res[str(arm)][0]["digest"] for arm in arms]
    summary = {}
    for arm in arms:
        rs = res[str(arm)]
        summary[str(arm)] = {k: {"median": statistics.median(x[k] for x in rs), "min": min(x[k] for x in rs), "max": max(x[k] for x in rs)}
                             for k in ("ms_match", "ms_score", "ms_gather")}
        summary[str(arm)]["pair_evaluations"] = rs[0]["pair_evaluations"]
        summary[str(arm)]["matches_after_knn"] = rs[0]["matches_after_knn"]
    out = {"workload": f"{VIEWS} views x {SEGS} segments, ring +-{RING}, synth seed {SEED}, kNN {KNN}, Line3D.matchImages",
           "gpu": gpus, "runs": a.runs, "arms": [str(arm) for arm in arms], "results": res, "summary": summary,
           "identical": all(d == digests[0] for d in digests)}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "multidevice.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps({"gpu": gpus, "summary": summary, "identical": out["identical"]}, indent=1))
    if not out["identical"]:
        sys.exit("the device lists gave different results")


if __name__ == "__main__":
    main()
