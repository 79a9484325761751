"""Geometry sweep of k_match_topk on the benchmark's workload (bench.py: 1000 views x 3000 segments, ring +-5).

    python tools/sweep_tiles.py build        # no GPU needed: compiles one libl3d_b200_<tag>.so per variant (in parallel)
    python tools/sweep_tiles.py run [OUT]    # on the GPU: bench.py per variant (base first and last), optional JSON to OUT
"""
import json, os, subprocess, sys
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
VARIANTS = {     # warps per CTA (one CTA per SM), row slots per warp, most rows per work unit, TMA ring depth (6 x 512: 3072 resident)
    "base_W24_S8_U1024": [],
    "U512": ["MK_UNIT_ROWS=512"],
    "U1536": ["MK_UNIT_ROWS=1536"],
    "U3072": ["MK_UNIT_ROWS=3072"],
    "S4": ["MK_SLOTS=4"],
    "W20": ["MK_WARPS=20"],
    "W16": ["MK_WARPS=16"],
}
if sys.argv[1] == "build":
    from line3dpp_b200 import build
    from concurrent.futures import ThreadPoolExecutor
    with ThreadPoolExecutor(len(VARIANTS)) as ex:
        for tag, path in zip(VARIANTS, ex.map(lambda kv: build.build(defines=kv[1], out=f"libl3d_b200_{kv[0]}.so"), VARIANTS.items())):
            print(tag, path, flush=True)
elif sys.argv[1] == "run":
    res = {}
    for tag in list(VARIANTS) + ["base_W24_S8_U1024"]:
        so = os.path.join(ROOT, "line3dpp_b200", f"libl3d_b200_{tag}.so")
        if not os.path.exists(so):
            continue
        env = dict(os.environ, L3D_LIB=so, L3D_BENCH_LEAN="1")
        out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", "5", "--warmup", "3"], env=env,
                             capture_output=True, text=True).stdout
        lines = [l for l in out.splitlines() if l.startswith("{")]
        ms = json.loads(lines[-1])["ms_per_step"] if lines else float("nan")
        res.setdefault(tag, []).append(ms)
        print(f"{tag:24s} {ms:.2f} ms per step", flush=True)
    if len(sys.argv) > 2:
        json.dump({"workload": "bench.py --gpus 1 --steps 5 --warmup 3", "ms_per_step": res}, open(sys.argv[2], "w"), indent=1)
