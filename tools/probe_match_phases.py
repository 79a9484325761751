"""Where the warps of k_match_topk spend their cycles, on the benchmark's workload (ring +-5, 3000 segments per view, kNN 10; the
first V views, 5 V view pairs).

    python tools/probe_match_phases.py build [O0]     # no GPU needed: line3dpp_b200/libl3d_b200_probe.so (-DL3D_MATCH_PROBE); O0:
                                                      # libl3d_b200_probe_O0.so, window pieces in class order (MK_SCAN_ORDER=0)
    python tools/probe_match_phases.py run [V]        # on the GPU (default V = 100); L3D_LIB=<.so> runs another probe build

The probe build adds clock64() spans per warp (l3d_match.cuh, MP_*); without the define none of it is compiled.  A row's set-up is three
phases: "setup" (setup_row: its constants), "window" (its window positions in every arc class) and "pieces" (their concatenation).  Shares are of all
warp-cycles of the launch: every warp's time from its first instruction to the end of its CTA.  "other" is the busy time no phase
covers (the CTA prologue before its barrier).  The spread compares, per CTA, the longest and the shortest warp busy time.  The
counters split the exact evaluations by the test that stops them (overlap, then depths) and count the keys pushed into row lists and
the prune_row calls that cut a full list to its k best.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))

PHASES = ["setup", "window", "pieces", "scan", "exact", "finalize", "wait", "tail"]
KEYS = PHASES + ["rows", "entries", "survivors", "evals", "drains", "overlap_pass", "depth_pass", "pushed", "prunes", "ctas", "busy_max",
                 "busy_min", "busy_sum"]
SO = "libl3d_b200_probe.so"


def run(V):
    import ctypes as C
    from line3dpp_b200 import capi, synth
    from tests import util
    os.environ.setdefault("L3D_LIB", os.path.join(os.path.dirname(capi.__file__), SO))
    sc = synth.make_scene(V, 3000, 1004, "ring5")
    pairs = synth.view_pairs(sc.neighbors)
    F = util.pair_F(sc, pairs)
    ctx = capi.Context(0)
    ctx.set_views(util.scene_descs(sc), sc.segs)
    out = np.zeros(len(KEYS), np.uint64)
    probe = capi.lib().l3d_match_probe
    ctx.match_pairs(pairs, F, 0.25, 10)                      # warm-up
    ctx.sync()
    assert probe(out.ctypes.data_as(C.c_void_p), 1) == len(KEYS)
    ctx.match_pairs(pairs, F, 0.25, 10)
    ctx.sync()
    assert probe(out.ctypes.data_as(C.c_void_p), 1) == len(KEYS)
    ctx.close()
    p = dict(zip(KEYS, out.astype(np.float64)))
    total = p["busy_sum"] + p["tail"]
    print(f"{os.path.basename(os.environ['L3D_LIB'])}: {len(pairs)} view pairs, {int(p['ctas'])} CTAs, {int(p['rows'])} row set-ups")
    print("| phase | share of warp-cycles |\n|---|---|")
    for k in PHASES:
        print(f"| {k} | {p[k] / total:.1%} |")
    print(f"| row set-up (setup + window + pieces) | {sum(p[k] for k in PHASES[:3]) / total:.1%} |")
    print(f"| other | {(p['busy_sum'] - sum(p[k] for k in PHASES[:-1])) / total:.1%} |")
    print(f"warp busy time inside a CTA, summed over CTAs: shortest / longest {p['busy_min'] / p['busy_max']:.3f}, "
          f"mean / longest {p['busy_sum'] / total:.3f}")
    rows = max(p["rows"], 1.0)
    print(f"per row set-up: {p['entries'] / rows:.1f} window entries, {p['survivors'] / rows:.1f} survivors of both filters, "
          f"{p['evals'] / rows:.1f} exact evaluations; early queue drains {int(p['drains'])}")
    ev = max(p["evals"], 1.0)
    print(f"exact evaluations {int(p['evals'])}: {int(p['overlap_pass'])} pass the overlap test ({p['overlap_pass'] / ev:.1%}, "
          f"{32 * p['overlap_pass'] / ev:.1f} of 32 lanes per batch), {int(p['depth_pass'])} the depth test too ({p['depth_pass'] / ev:.1%}); "
          f"{int(p['pushed'])} keys pushed, {int(p['prunes'])} prune_row calls ({p['prunes'] / rows:.2f} per row)")


if __name__ == "__main__":
    if sys.argv[1] == "build":
        from line3dpp_b200 import build
        o0 = sys.argv[2:] == ["O0"]
        print(build.build(defines=["L3D_MATCH_PROBE"] + (["MK_SCAN_ORDER=0"] if o0 else []), out=SO.replace(".so", "_O0.so") if o0 else SO))
    elif sys.argv[1] == "run":
        run(int(sys.argv[2]) if len(sys.argv) > 2 else 100)
