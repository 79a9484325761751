"""Geometry sweep of k_match_topk on the benchmark's workload (bench.py: 1000 views x 3000 segments, ring +-5).

    python tools/sweep_tiles.py build [TAG ...]              # no GPU needed: compiles one libl3d_b200_<tag>.so per variant (in parallel)
    python tools/sweep_tiles.py run [OUT.json] [--reps N] [TAG ...]  # on the GPU: bench.py per variant, N rounds over the variants
                                                                     # with the base first and last, optional JSON to OUT.json
TAG ...: only these variants (the base is always run).  Interleaved rounds in one session keep clock and host drift out of the
comparison.
"""
import json, os, subprocess, sys
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
BASE = "base"
# warps per CTA (one CTA per SM), row slots per warp, most rows per work unit, TMA ring depth (6 x 512: 3072 resident), keys per row
# before the first prune, order of a row's window pieces; the base is l3d_match.cuh's default: 32 warps x 8 slots, 1024-row units,
# 32 keys, nearest arc class first
VARIANTS = {
    BASE: [],
    "U512": ["MK_UNIT_ROWS=512"],
    "U1536": ["MK_UNIT_ROWS=1536"],
    "U3072": ["MK_UNIT_ROWS=3072"],
    "S4": ["MK_SLOTS=4"],
    "W20": ["MK_WARPS=20"],
    "W16": ["MK_WARPS=16"],
    "W24": ["MK_WARPS=24"],
    "W28": ["MK_WARPS=28"],
    "C16": ["MK_CAP=16"],
    "C24": ["MK_CAP=24"],
    "O0": ["MK_SCAN_ORDER=0"],
}
args = sys.argv[2:]
reps = 1
if "--reps" in args:
    i = args.index("--reps")
    reps = int(args[i + 1])
    del args[i:i + 2]
out_json = args.pop(0) if sys.argv[1] == "run" and args and args[0].endswith(".json") else None
tags = [BASE] + [t for t in args if t != BASE] if args else list(VARIANTS)
if sys.argv[1] == "build":
    from line3dpp_b200 import build
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(len(tags)) as ex:
        for tag, path in zip(tags, ex.map(lambda t: build.build(defines=VARIANTS[t], out=f"libl3d_b200_{t}.so"), tags)):
            print(tag, path, flush=True)
elif sys.argv[1] == "run":
    res = {}
    for tag in tags * reps + [BASE]:
        so = os.path.join(ROOT, "line3dpp_b200", f"libl3d_b200_{tag}.so")
        if not os.path.exists(so):
            continue
        env = dict(os.environ, L3D_LIB=so, L3D_BENCH_LEAN="1")
        out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", "5", "--warmup", "3"], env=env,
                             capture_output=True, text=True).stdout
        lines = [l for l in out.splitlines() if l.startswith("{")]
        line = json.loads(lines[-1]) if lines else {}
        ms = line.get("ms_per_step", float("nan"))
        res.setdefault(tag, []).append(ms)
        print(f"{tag:12s} {ms:.2f} ms per step  clocks {line.get('clocks')}", flush=True)
    if out_json:
        json.dump({"workload": "bench.py --gpus 1 --steps 5 --warmup 3", "ms_per_step": res}, open(out_json, "w"), indent=1)
