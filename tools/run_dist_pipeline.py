"""The whole hot path through L3DPP::Line3D on N GPUs (one process per GPU, NCCL): matching sharded over the view pairs
(Line3D::setShard, line3dpp_b200/dist.py), match rows broadcast in place, scoring sweep / affinity / diffusion / clustering
replicated.  Prints ONE JSON line on rank 0: stage timings (max over ranks), per-rank HBM high-water, and a digest check that
every rank ended with the same result; `--check-views K` also runs the first K views sharded AND unsharded and compares them
bit for bit (multi-GPU == single-GPU).  `--knn` is matchImages' kNN; keep-all (<= 0) and > 32 exchange twice (counts, then the
rows at the stride the counts give), and the line reports both times (ms_exchange_counts_max, ms_exchange_records_max), the record
array every rank ends up holding, which is what the exchange moves in all (record_array_bytes = rows x record_stride x 24 B; for
keep-all one GPU, where nothing is exchanged, holds the same array) and, for comparison, the bytes of the matches themselves (match_record_bytes =
matches_after_knn x 24 B).

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P \
        tools/run_dist_pipeline.py --views 1000 --segs 3000 --ring 5 --diffusion 1 [--knn 10] [--check-views 60] [--reps 2]
"""
import argparse
import hashlib
import json
import os
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from line3dpp_b200 import line3d, synth, dist as l3dist   # noqa: E402


def digest(L, cams):
    b, p = L.estimates()
    s, r = L.segments3d(), L.residuals()
    h = hashlib.sha256()
    for a in (b, p, s, r):
        h.update(a.tobytes())
    for c in cams:
        h.update(L.view_matches(c, True).tobytes())
    return h.hexdigest()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", type=int, default=1000)
    ap.add_argument("--segs", type=int, default=3000)
    ap.add_argument("--ring", type=int, default=5)
    ap.add_argument("--diffusion", type=int, default=1)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--check-views", type=int, default=0)
    ap.add_argument("--seed", type=int, default=1004)
    ap.add_argument("--knn", type=int, default=10)
    a = ap.parse_args()
    rank, dev, world = int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    torch.cuda.set_device(dev)
    # rank 0 prints ONE JSON line: the "NCCL version ..." banner goes to stdout unless NCCL's log is pointed elsewhere (measured on the
    # 2-GPU box: banner with NCCL_DEBUG unset, none with NCCL_DEBUG=WARN + NCCL_DEBUG_FILE=/dev/stderr)
    os.environ.setdefault("NCCL_DEBUG", "WARN")
    os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", dev))
    out = {"views": a.views, "segments_per_view": a.segs, "ring": a.ring, "n_gpus": world, "diffusion": bool(a.diffusion), "knn": a.knn}
    free0, total_mem = torch.cuda.mem_get_info()

    # ---- optional bit check on a sub-ring: sharded == unsharded
    if a.check_views:
        sc = synth.make_scene(a.check_views, a.segs, a.seed + 1, f"ring{a.ring}")
        full = line3d.Line3D(neighbors_by_worldpoints=False, device=dev)
        full.add_scene(sc); full.match_images(knn=a.knn); full.reconstruct_3d_lines(3, bool(a.diffusion))
        want = digest(full, sc.cam_ids[:8])
        nl = full.stats()["lines3D"]
        full.close()
        L = line3d.Line3D(neighbors_by_worldpoints=False, device=dev)
        L.add_scene(sc)
        if world > 1:
            keep = l3dist.attach(L, dev)   # noqa: F841
        L.match_images(knn=a.knn); L.reconstruct_3d_lines(3, bool(a.diffusion))
        ok = digest(L, sc.cam_ids[:8]) == want
        L.close()
        t = torch.tensor([1 if ok else 0], device="cuda")
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MIN)
        out["check"] = {"views": a.check_views, "lines3D": nl, "sharded_equals_unsharded_on_every_rank": bool(t.item())}
        torch.cuda.empty_cache()

    t0 = time.time()
    sc = synth.make_scene(a.views, a.segs, a.seed, f"ring{a.ring}")
    out["scene_s"] = time.time() - t0
    L = line3d.Line3D(neighbors_by_worldpoints=False, device=dev)
    t0 = time.time(); L.add_scene(sc); out["add_s"] = time.time() - t0
    if world > 1:
        keep = l3dist.attach(L, dev)   # noqa: F841
    best, calls = None, []
    for rep in range(a.reps):
        if world > 1:
            dist.barrier()
            L._exchange_state["exchanges"].clear()
        torch.cuda.synchronize()
        t0 = time.time(); L.match_images(knn=a.knn); torch.cuda.synchronize(); t_match = time.time() - t0
        t0 = time.time(); L.reconstruct_3d_lines(3, bool(a.diffusion)); torch.cuda.synchronize(); t_rec = time.time() - t0
        st = L.stats()
        calls = list(L._exchange_state["exchanges"]) if world > 1 else []
        counts_ms = sum(c["ms"] for c in calls if c["knn"] == 0)
        records_ms = sum(c["ms"] for c in calls if c["knn"] > 0)
        cur = dict(matchImages_s=t_match, reconstruct_s=t_rec, ms_match_incl_exchange=st["ms_match"], ms_exchange=counts_ms + records_ms,
                   ms_exchange_counts=counts_ms, ms_exchange_records=records_ms, ms_score=st["ms_score"],
                   ms_affinity=st["ms_affinity"], ms_diffusion=st["ms_diffusion"], ms_cluster=st["ms_cluster"])
        if best is None or cur["matchImages_s"] + cur["reconstruct_s"] < best["matchImages_s"] + best["reconstruct_s"]:
            best = cur
    st = L.stats()
    stride, rows = int(L.L.l3d_match_stride(L.ctx)), int(L.L.l3d_match_total_rows(L.ctx))
    free1, _ = torch.cuda.mem_get_info()
    keys = sorted(best)
    t = torch.tensor([best[k] for k in keys] + [float(total_mem - free1), float(st["pair_evaluations"])], dtype=torch.float64, device="cuda")
    dg = digest(L, sc.cam_ids[:4])
    dgt = torch.tensor(list(bytes.fromhex(dg)), dtype=torch.uint8, device="cuda")
    if world > 1:
        tmax = t.clone(); dist.all_reduce(tmax, op=dist.ReduceOp.MAX)
        tsum = t.clone(); dist.all_reduce(tsum, op=dist.ReduceOp.SUM)
        allmem = [torch.zeros_like(t) for _ in range(world)]; dist.all_gather(allmem, t)
        alld = [torch.zeros_like(dgt) for _ in range(world)]; dist.all_gather(alld, dgt)
        same = all(bool((d == dgt).all().item()) for d in alld)
    else:
        tmax, tsum, allmem, same = t, t, [t], True
    if rank == 0:
        for i, k in enumerate(keys):
            out[k + "_max"] = tmax[i].item()
        out["hbm_used_gb_per_rank"] = [round(m[len(keys)].item() / 1e9, 2) for m in allmem]
        out["pair_evaluations_per_rank"] = [int(m[len(keys) + 1].item()) for m in allmem]
        out["pair_evaluations"] = int(tsum[len(keys) + 1].item())
        out["pair_evals_per_s_matchImages"] = out["pair_evaluations"] / out["matchImages_s_max"]
        out["identical_result_on_every_rank"] = same
        for k in ("view_pairs", "matches_after_knn", "estimates", "affinity_entries", "affinity_rows", "clusters_valid", "lines3D"):
            out[k] = st[k]
        out["exchange_calls"] = len(calls)
        out["record_stride"] = stride
        out["record_array_bytes"] = 24 * rows * stride
        out["match_record_bytes"] = 24 * st["matches_after_knn"]
        print(json.dumps(out))
    L.close()
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
