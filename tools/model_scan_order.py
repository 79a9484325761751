"""CPU model of how many candidates of a row reach k_match_topk's exact path, for the two orders in which a row can scan its window
pieces (MK_SCAN_ORDER, l3d_match.cuh): class order 0 .. NCLS - 1, or the arc class nearest the row's own span first.  numpy only.

    python tools/model_scan_order.py [PAIRS] [STRIDE]     # default: 3 view pairs of the benchmark's scene, every 3rd source row

The scene is the benchmark's (bench.py: 1000 views x 3000 segments, seed 1004, ring +-5); only the views of the modelled pairs are
materialised.  Per target the model takes the kernel's arc class and arc start (tests/level1_model.py, the numpy restatement of the
level-1 tables); targets without an arc come last, as the kernel scans them.  Per row it takes the span class of its two kappa values.
What it models: a candidate is queued when its overlap passes the float filter's 0.95 x score-to-beat (less a 0.03 margin for the
filter's conservatism), the queue is evaluated 32 at a time against the score-to-beat of the batch's start, a row's list holds 32 keys
and is cut to its k best when a 33rd arrives.  What it does not: the level-1 arc test (only the window order), the filter's exact
margins, and the queue that the rows of a warp share.  The overlap is the reference's inner / outer in double.
"""
import os
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
from line3dpp_b200 import synth            # noqa: E402
from tests import level1_model as l1       # noqa: E402

EPI, K, CAP, BATCH = 0.25, 10, 32, 32
EXT = 1.0 / EPI + 0.5                      # extension of a target arc at this epi_overlap (build_level1, l3d_capi.cu)
VIEWS, SEGS, SEED, RING = 1000, 3000, 1004, 5


def overlaps(F, S, T):
    """overlap[row, target]: both source endpoints' epipolar lines cut the target line at t1, t2 (t = 0 / 1 at its endpoints)"""
    h = lambda P: np.c_[P, np.ones(len(P))]
    e1, e2 = h(S[:, 0:2]) @ F.T, h(S[:, 2:4]) @ F.T
    q1, q2 = h(T[:, 0:2]), h(T[:, 2:4])
    with np.errstate(all="ignore"):
        t1 = (e1 @ q1.T) / (e1 @ q1.T - e1 @ q2.T)
        t2 = (e2 @ q1.T) / (e2 @ q1.T - e2 @ q2.T)
        lo, hi = np.minimum(t1, t2), np.maximum(t1, t2)
        inner = np.minimum(hi, 1.0) - np.maximum(lo, 0.0)
        outer = np.maximum(hi, 1.0) - np.minimum(lo, 0.0)
        return np.nan_to_num(np.where(inner > 0.0, inner / outer, 0.0))


def exact_evals(ov_row, order):
    """exact evaluations of one row whose filter survivors arrive in `order`"""
    thr_s, row_thr, keys, queue, evals = 0.95 * EPI, 0.0, [], [], 0
    for n, j in enumerate(order):
        if ov_row[j] > thr_s - 0.03:
            queue.append(j)
        if len(queue) == BATCH or (n == len(order) - 1 and queue):
            evals += len(queue)
            kept = [ov_row[q] for q in queue if ov_row[q] > EPI and ov_row[q] >= row_thr]
            for o in kept:
                if len(keys) == CAP:
                    keys = sorted(keys, reverse=True)[:K]
                    row_thr = keys[-1]
                    thr_s = 0.95 * max(row_thr, EPI)
                keys.append(o)
            queue = []
    return evals


def main(npairs=3, stride=3):
    pairs = synth.view_pairs(synth.ring_neighbors(VIEWS, RING))[:npairs]
    sc = synth.make_scene_views(VIEWS, SEGS, SEED, f"ring{RING}", sorted({int(v) for p in pairs for v in p}))
    tot = {"class order (MK_SCAN_ORDER=0)": [], "nearest class first (MK_SCAN_ORDER=1)": []}
    for s, t in pairs:
        F = synth.fundamental(sc.K[s], sc.R[s], sc.t[s], sc.K[t], sc.R[t], sc.t[t])
        Ff = F.astype(np.float32)
        u, v, _ = l1.basis(Ff)
        S, T = sc.segs[s].astype(np.float64), sc.segs[t].astype(np.float64)
        ov = overlaps(F, S, T)
        cls, start = np.empty(len(T), int), np.zeros(len(T), np.int64)
        for j, q in enumerate(sc.segs[t]):
            arc = l1.target_arc(u, v, q, EXT)
            cls[j] = l1.NCLS if arc is None else l1.arc_class(arc[1])
            start[j] = 0 if arc is None else arc[0]
        base = np.lexsort((np.arange(len(T)), start, cls))       # class, then arc start: the level-1 table's order
        for r in range(0, len(S), stride):
            k1, _ = l1.line_kappa(u, v, l1.epipolar_line(Ff, *sc.segs[s][r, 0:2]))
            k2, _ = l1.line_kappa(u, v, l1.epipolar_line(Ff, *sc.segs[s][r, 2:4]))
            span = min((k2 - k1) & l1.M32, (k1 - k2) & l1.M32)
            rc = min(l1.arc_class(span), l1.NCLS - 1)
            cand = base[ov[r, base] > 0.0]
            c = cls[cand]
            dist = np.where(c == l1.NCLS, 2 * l1.NCLS, np.abs(c - rc))
            near = cand[np.lexsort((np.arange(len(cand)), c, dist))]   # stable: arc start order inside a class
            for name, order in zip(tot, (cand, near)):
                tot[name].append(exact_evals(ov[r], order))
    rows = len(next(iter(tot.values())))
    print(f"{len(pairs)} view pairs of the benchmark's scene, {rows} rows (every {stride}. row), kNN {K}, epi_overlap {EPI}")
    means = {k: float(np.mean(v)) for k, v in tot.items()}
    for k, m in means.items():
        print(f"{k:40s} {m:6.1f} exact evaluations per row")
    a, b = means.values()
    print(f"change {100.0 * (b - a) / a:+.1f} %")


if __name__ == "__main__":
    main(*(int(a) for a in sys.argv[1:3]))
