"""Device time of matching against caller-given candidates (l3d_match_pairs_cand) next to the epipolar scan of the same pairs.

    python tools/bench_candidates.py --out DIR [--pairs 200] [--iters 5]

Workload: the views of BASELINE.json configs[3] (3000 segments per view, ring +-5 neighbours, synth seed 1003, kNN 10) and the first
`pairs` view pairs of its pair list, all restricted.  Each source row gets c = 4, 16 and 64 candidates: its true top-k (the scan's
emitted matches, at most c of them) and random targets for the rest, built on the device and passed as a device array.
Whole calls: per arm and iteration the L2 is flushed (a 256 MB write), then CUDA events on the context's stream and the host clock
time one call, everything included: for a restricted call the read-back of the device triples, their check on the host, the upload of
the pair tables, the kernels and the wait for the distinct count.  The SM clock and power draw are sampled (nvidia-smi, every 100 ms)
while those calls run.  Kernels: one more call per iteration runs under torch.profiler (CUPTI), and the kernel times are summed by phase:
  sort  = every kernel of a restricted call but k_match_cand: k_cand_keys and cub's radix sort and unique kernels
  match = k_match_cand
  scan  = every kernel of l3d_match_pairs_range over the same pairs (level-1 tables, row windows, k_match_topk)
Kernel boundaries inside one C call are not visible to events recorded around it, hence the profiler for the split.  Reported: medians
over the iterations, candidate evaluations per second (distinct candidates / match time) and the scan's cells per second.  The card
name, power limit and maximum SM clock are read in the same run (queries only).  Writes DIR/candidates.json.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

VIEWS, SEGS, SEED, RING, KNN = 1000, 3000, 1003, 5, 10


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines() if r.returncode == 0 else ["nvidia-smi failed"]
    except (OSError, subprocess.SubprocessError):
        return ["nvidia-smi unavailable"]


def phase(name):
    return "match" if "k_match_cand" in name else "sort"


class ClockSampler:
    """nvidia-smi's SM clock and power draw every 100 ms while the block runs (a query; the process ends with the block)"""

    def __enter__(self):
        dev = (os.environ.get("CUDA_VISIBLE_DEVICES") or "0").split(",")[0]
        try:
            self.p = subprocess.Popen(["nvidia-smi", "-i", dev, "--query-gpu=clocks.sm,power.draw", "--format=csv,noheader,nounits", "-lms", "100"],
                                      stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
        except OSError:
            self.p = None
        self.samples = []
        return self

    def __exit__(self, *exc):
        if self.p is None:
            return False
        self.p.terminate()
        try:
            out, _ = self.p.communicate(timeout=10)
        except subprocess.TimeoutExpired:
            self.p.kill()
            out, _ = self.p.communicate()
        for line in out.splitlines():
            try:
                clk, pw = (float(x) for x in line.split(","))
                self.samples.append((clk, pw))
            except ValueError:
                pass
        return False

    def summary(self):
        if not self.samples:
            return {"sm_clock_mhz": None, "power_w": None}
        return {"sm_clock_mhz": statistics.median(c for c, _ in self.samples), "power_w": statistics.median(p for _, p in self.samples),
                "samples": len(self.samples)}


def timed_calls(fn, flush, stream, iters):
    """(median event ms, median wall ms) of at least `iters` whole calls and at least 1.5 s of them (so that the sampler sees the clocks
    under load), each after an L2 flush, and the clocks seen meanwhile"""
    import torch
    ev, wall = [], []
    with ClockSampler() as clk:
        start = time.perf_counter()
        while len(ev) < iters or time.perf_counter() - start < 1.5:
            flush.zero_()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0 = time.perf_counter()
            e0.record(stream)
            fn()
            e1.record(stream)
            torch.cuda.synchronize()
            wall.append((time.perf_counter() - t0) * 1e3)
            ev.append(e0.elapsed_time(e1))
    return statistics.median(ev), statistics.median(wall), clk.summary()


def profiled(fn, flush):
    import torch
    from torch.profiler import ProfilerActivity, profile
    flush.zero_()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.events():
        if e.device_type.name == "CUDA" and e.device_time_total > 0 and "memset" not in e.name.lower() and "memcpy" not in e.name.lower():
            k = phase(e.name)
            out[k] = out.get(k, 0.0) + e.device_time_total / 1000.0
            out["all"] = out.get("all", 0.0) + e.device_time_total / 1000.0
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--pairs", type=int, default=200)
    ap.add_argument("--iters", type=int, default=5)
    args = ap.parse_args()
    import numpy as np
    import torch
    from line3dpp_b200 import capi, synth
    from tests import util

    if not torch.cuda.is_available():
        raise SystemExit("bench_candidates needs a CUDA device (no CPU fallback)")
    info = gpu_info()
    sc = synth.make_scene(VIEWS, SEGS, SEED, f"ring{RING}")
    pairs = np.ascontiguousarray(synth.view_pairs(sc.neighbors, sc.cam_ids)[:args.pairs], np.int32)
    ctx = capi.Context(0)
    ctx.set_views(util.scene_descs(sc), sc.segs)
    F = util.pair_F(sc, pairs)
    flush = torch.empty(64 << 20, dtype=torch.float32, device="cuda")
    stream = torch.cuda.ExternalStream(ctx.stream)
    # the scan: its emitted top-k per row are every row's true candidates
    ctx.match_pairs_range(pairs, F, 0, len(pairs), 0.25, KNN)
    row_ptr, recs = ctx.matches_csr()
    cells = int(sum(len(sc.segs[s]) * len(sc.segs[t]) for s, t in pairs))
    rows = len(row_ptr) - 1
    pair_of_row = np.repeat(np.arange(len(pairs)), [len(sc.segs[s]) for s, _ in pairs]).astype(np.int32)
    src_of_row = np.concatenate([np.arange(len(sc.segs[s])) for s, _ in pairs]).astype(np.int32)
    nt_of_row = np.array([len(sc.segs[t]) for _, t in pairs], np.int64)[pair_of_row]
    counts = np.diff(row_ptr)
    g = torch.Generator(device="cuda").manual_seed(7)
    result = {"gpu": info, "pairs": len(pairs), "rows": rows, "scan_cells": cells, "knn": KNN, "arms": {}}
    scan_call = lambda: ctx.match_pairs_range(pairs, F, 0, len(pairs), 0.25, KNN)
    scan = [profiled(scan_call, flush) for _ in range(args.iters + 1)][1:]
    result["scan_ms"] = statistics.median(s["all"] for s in scan)
    result["scan_cells_per_s"] = cells / (result["scan_ms"] / 1e3)
    result["scan_call_event_ms"], result["scan_call_wall_ms"], result["scan_clocks"] = timed_calls(scan_call, flush, stream, 2 * args.iters)
    result["scan_matches"] = int(recs.shape[0])
    prow = torch.from_numpy(pair_of_row).cuda(); srow = torch.from_numpy(src_of_row).cuda(); ntr = torch.from_numpy(nt_of_row).cuda()
    cnt = torch.from_numpy(counts).cuda(); rp = torch.from_numpy(row_ptr[:-1]).cuda()
    tgt_all = torch.from_numpy(recs["tgt_seg"].astype(np.int64)).cuda()
    for c in (4, 16, 64):
        col = torch.arange(c, device="cuda")
        rand = (torch.rand((rows, c), generator=g, device="cuda") * ntr[:, None]).long()
        true_idx = (rp[:, None] + col[None, :]).clamp(max=max(len(tgt_all) - 1, 0))
        is_true = col[None, :] < cnt[:, None]
        tgt = torch.where(is_true, tgt_all[true_idx] if len(tgt_all) else rand, rand)
        trip = torch.stack([prow[:, None].expand(rows, c), srow[:, None].expand(rows, c), tgt], -1).reshape(-1, 3).to(torch.int32).contiguous()
        torch.cuda.synchronize()
        run = lambda: ctx.match_pairs_cand(pairs, F, np.ones(len(pairs), np.int32), (trip.data_ptr(), trip.shape[0]), 0.25, KNN, on_device=True)
        t = [profiled(run, flush) for _ in range(args.iters + 1)][1:]
        ev_ms, wall_ms, clocks = timed_calls(run, flush, stream, 2 * args.iters)
        distinct = ctx.match_pair_evals()
        _, crecs = ctx.matches_csr()
        sort_ms, match_ms = statistics.median(x.get("sort", 0.0) for x in t), statistics.median(x.get("match", 0.0) for x in t)
        result["arms"][str(c)] = {"triples": int(trip.shape[0]), "distinct": int(distinct), "sort_ms": sort_ms, "match_ms": match_ms,
                                  "all_kernels_ms": statistics.median(x["all"] for x in t), "evals_per_s": distinct / (match_ms / 1e3),
                                  "matches": int(crecs.shape[0]), "call_event_ms": ev_ms, "call_wall_ms": wall_ms, "clocks": clocks}
        del trip, rand, tgt
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "candidates.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result, indent=1))
    ctx.close()


if __name__ == "__main__":
    main()
