"""Float64 restatement of computingAffinityMatrix (line3D.cc:1852-2023), written from the reference's sequential loop and
independently of oracle/l3d_oracle.cc and csrc/l3d_affinity.cu (no pair sort, no fixpoint, no atomic minima).

  * similarity() is Line3D::similarity (line3D.cc:1467-1553, truncate = false) in float64, vectorised over every query the loop
    can make: 0 without an estimate or for a segment shorter than L3D_EPS; the dot product of the directions clamped to [-1, 1]
    and the angle folded above 90 degrees; the cutoff depths min(median_depth, med_scene_depth_lines) only when the latter is
    above L3D_EPS; sigma = cutoff * k where a depth exceeds its cutoff, depth * k otherwise; fmin that ignores NaN (a zero
    regulariser with a zero distance is 0 / 0).
  * The loop (restate) walks the estimates in (camID, segment) order and each one's kept matches in list order with a `used` set of
    unordered pairs (unused(), 1982-2002), a first-come local-id map (getLocalID, 2005-2023) and found_aff: the direct edge
    (1881-1900), the links through its target only if that edge was new (1904-1937), the links through the source only if some
    direct edge of the segment was new (1941-1974).

restate() also returns the superset candidate list that l3d_affinity_edges emits (every event whose own similarity passes and
whose parent's passes, in emission order), a counter of the paths the problem reaches, the longest dependency chain and the number
of similarities within GUARD of min_affinity.  The scene builders at the end derive scenes from synth.make_scene(collinear=True)
that reach every path the loop has."""
import collections
import dataclasses

import numpy as np

EPS = 1e-12                       # L3D_EPS
GUARD = 1e-5                      # a similarity this close to min_affinity could pass in float64 and fail in float32 (or back)

# the paths restate() counts (hits[...]); "a_by_b": an event of kind a that unused() rejected because an earlier event of kind b
# took its pair.  direct / tlink pairs span two views and a source link pair lies within one, so slink_by_direct, slink_by_tlink,
# direct_by_slink and tlink_by_slink cannot happen (counted anyway, so that a test can assert they stay 0).
PATHS = ("direct_by_direct", "direct_by_tlink", "direct_by_slink", "tlink_by_direct", "tlink_by_tlink", "tlink_by_slink",
         "slink_by_direct", "slink_by_tlink", "slink_by_slink",
         "tlink_skipped",          # a link through the target whose similarity passes, not tried: its direct edge was rejected
         "slink_gated",            # a link through the source whose similarity passes, not tried: a kept match passed, none was new
         "slink_after_failed",     # source links tried after the segment's last kept match failed
         "id_by_tlink", "id_by_slink",   # a local id first assigned to the target of a link
         "partner_no_estimate",    # a collinear partner without an estimate
         "angle_gt_90", "depth_gt_cutoff", "depth_le_cutoff", "no_scene_cutoff")


@dataclasses.dataclass
class Problem:
    """what computingAffinityMatrix reads.  Segments are (camID, segment id) tuples.
    est_cam, est_seg, est_d1, est_d2: the best match of every estimate (src cam / seg, depth_p1 / depth_p2), any order;
    est_P [E, 6]: its P1, P2.  kept[(cam, seg)]: the kept matches of a segment as target segments, in list order.
    collin[(cam, seg)]: its collinear segment ids (None: links off).  views[cam] = (k, median_depth)."""
    est_cam: np.ndarray
    est_seg: np.ndarray
    est_d1: np.ndarray
    est_d2: np.ndarray
    est_P: np.ndarray
    kept: dict
    collin: dict | None
    views: dict


@dataclasses.dataclass
class Result:
    ei: np.ndarray                # the CLEdge list A_: (id1, id2, w), (id2, id1, w) per accepted edge
    ej: np.ndarray
    ew: np.ndarray                # float64
    l2g: list                     # local id -> segment
    cand: list                    # (segment, segment, w) superset candidates in emission order
    acc: np.ndarray               # the candidate behind every accepted edge (an index into cand)
    hits: collections.Counter
    chain: int                    # longest dependency chain
    band: int                     # similarities within GUARD of min_affinity that `decided` does not settle
    near: set                     # the (segment, segment) queries whose similarity lies within GUARD of min_affinity


def problem(best, P, matches, collin, views):
    """a Problem from exported arrays: best = the estimates' best matches (fields src_cam, src_seg, d_p1, d_p2), P [E, 6];
    matches = the kept matches of every view (fields src_cam, src_seg, tgt_cam, tgt_seg), each segment's in list order;
    collin = {cam: (row_ptr, idx)} (None: links off); views = {cam: (k, median_depth)}"""
    kept = {}
    for m in matches:
        for sc, ss, tc, ts in zip(*(m[f].tolist() for f in ("src_cam", "src_seg", "tgt_cam", "tgt_seg"))):
            kept.setdefault((sc, ss), []).append((tc, ts))
    col = None
    if collin is not None:
        col = {}
        for cam, (rp, idx) in collin.items():
            for s in np.flatnonzero(np.diff(rp)).tolist():
                col[(int(cam), s)] = idx[rp[s]:rp[s + 1]].tolist()
    return Problem(best["src_cam"].astype(np.int64), best["src_seg"].astype(np.int64), np.asarray(best["d_p1"]), np.asarray(best["d_p2"]),
                   np.asarray(P, np.float64), kept, col, {int(c): (float(k), float(md)) for c, (k, md) in views.items()})


def similarities(pr, a, b, two_sigA_sqr, med_scene_depth_lines):
    """similarity() of estimate a with the estimate b (-1: none) for index arrays a, b; also returns the path flags of each query
    (angle > 90, depth above / at or below its cutoff) as a dict of boolean arrays"""
    a, b = np.asarray(a, np.int64), np.asarray(b, np.int64)
    has = b >= 0
    bb = np.where(has, b, 0)
    P1, P2 = pr.est_P[:, :3], pr.est_P[:, 3:]
    L = np.linalg.norm(P2 - P1, axis=1)
    D = (P2 - P1) / np.where(L > EPS, L, 1.0)[:, None]
    k = np.array([pr.views[int(c)][0] for c in pr.est_cam], np.float64)
    md = np.array([pr.views[int(c)][1] for c in pr.est_cam], np.float64)
    c1, c2 = md[a], md[bb]
    if med_scene_depth_lines > EPS:
        c1, c2 = np.minimum(c1, med_scene_depth_lines), np.minimum(c2, med_scene_depth_lines)
    dot = np.clip((D[a] * D[bb]).sum(1), -1.0, 1.0)
    raw = np.degrees(np.arccos(dot))
    ang = np.where(raw > 90.0, 180.0 - raw, raw)
    sim_a = np.exp(-ang * ang / two_sigA_sqr)

    def dist(p, q1, dq):             # distance of point p from the line through q1 with direction dq
        h = q1 + dq * ((p - q1) * dq).sum(1, keepdims=True)
        return np.linalg.norm(h - p, axis=1)

    def term(d, dep, c, kk):
        sig = np.where(dep > c, c, dep) * kk
        reg = 2.0 * sig * sig
        with np.errstate(divide="ignore", invalid="ignore"):
            return np.exp(-d * d / reg)

    d1a, d2a, d1b, d2b = pr.est_d1[a].astype(np.float64), pr.est_d2[a].astype(np.float64), pr.est_d1[bb].astype(np.float64), pr.est_d2[bb].astype(np.float64)
    sp1 = np.fmin(term(dist(P1[a], P1[bb], D[bb]), d1a, c1, k[a]), term(dist(P2[a], P1[bb], D[bb]), d2a, c1, k[a]))
    sp2 = np.fmin(term(dist(P1[bb], P1[a], D[a]), d1b, c2, k[bb]), term(dist(P2[bb], P1[a], D[a]), d2b, c2, k[bb]))
    sim = np.fmin(sim_a, np.fmin(sp1, sp2))
    ok = has & (L[a] >= EPS) & (L[bb] >= EPS)
    flags = {"angle_gt_90": ok & (raw > 90.0),
             "depth_gt_cutoff": ok & ((d1a > c1) | (d2a > c1) | (d1b > c2) | (d2b > c2)),
             "depth_le_cutoff": ok & ((d1a <= c1) | (d2a <= c1) | (d1b <= c2) | (d2b <= c2))}
    return np.where(ok, sim, 0.0), flags


def restate(pr, two_sigA_sqr, med_scene_depth_lines, min_affinity, decided=None):
    """computingAffinityMatrix on problem pr (see the module docstring); returns a Result.  decided: {(segment, segment): passes}
    for similarities within GUARD of min_affinity, taken from elsewhere; band counts the ones it does not decide."""
    order = np.lexsort((pr.est_seg, pr.est_cam))                       # estimated_position3D_ order: camID, then segment
    seg_of = [(int(pr.est_cam[i]), int(pr.est_seg[i])) for i in order]
    entry = {s: int(i) for s, i in zip(seg_of, order)}                 # entry_map_
    seg_of_est = {i: s for s, i in entry.items()}
    col = pr.collin if pr.collin is not None else {}

    # every query the loop can make, so that the similarities are computed in one vectorised pass
    qa, qb, qseg, plan = [], [], [], []
    def query(i, t):
        qa.append(i); qb.append(entry.get(t, -1)); qseg.append((seg_of_est[i], t))
        return len(qa) - 1
    for s, i in zip(seg_of, order):
        direct = []
        for t in pr.kept.get(s, ()):
            t = (int(t[0]), int(t[1]))
            direct.append((t, query(i, t), [((t[0], c), query(i, (t[0], c))) for c in col.get(t, ())]))
        plan.append((s, direct, [((s[0], c), query(i, (s[0], c))) for c in col.get(s, ())]))
    sim, flags = similarities(pr, np.array(qa, np.int64), np.array(qb, np.int64), two_sigA_sqr, med_scene_depth_lines)
    sim = sim.tolist()

    hits = collections.Counter({p: 0 for p in PATHS})
    for f, v in flags.items():
        hits[f] = int(v.sum())
    if med_scene_depth_lines <= EPS:
        hits["no_scene_cutoff"] = len(qa)
    decided = decided or {}
    near = {q: decided.get(qseg[q]) for q in np.flatnonzero(np.abs(np.array(sim) - min_affinity) < GUARD).tolist()}
    band = sum(v is None for v in near.values())
    passes = lambda q: sim[q] > min_affinity if near.get(q) is None else near[q]

    used = {}                          # unordered pair -> kind of the event that took it
    last_chain = {}                    # unordered pair -> chain length of the last attempted event of the pair
    l2g, g2l, A, cand, acc = [], {}, [], [], []
    chain = 0

    def local_id(seg):
        if seg not in g2l:
            g2l[seg] = len(l2g); l2g.append(seg)
        return g2l[seg]

    def attempt(a, b, kind, parent_chain):
        """unused(a, b) for an event of `kind`; returns (new?, its chain length)"""
        nonlocal chain
        key = (min(a, b), max(a, b))
        c = 1 + max(parent_chain, last_chain.get(key, 0))
        last_chain[key] = c
        chain = max(chain, c)
        if key in used:
            hits[f"{kind}_by_{used[key]}"] += 1
            return False, c
        used[key] = kind
        return True, c

    def emit(lst, s):
        """the candidates of the links in lst that pass; returns the candidate index of each entry (-1: fails)"""
        idx = []
        for t2, q in lst:
            idx.append(len(cand) if passes(q) else -1)
            if passes(q):
                cand.append((s, t2, sim[q]))
        return idx

    def links(s, id1, lst, idx, kind, parent_chain):
        for (t2, q), ci in zip(lst, idx):
            if qb[q] < 0:
                hits["partner_no_estimate"] += 1
            if ci >= 0:
                ok, _ = attempt(s, t2, kind, parent_chain)
                if ok:
                    if t2 not in g2l:
                        hits[f"id_by_{kind}"] += 1
                    A.append((id1, local_id(t2), sim[q])); acc.append(ci)

    for s, direct, src_links in plan:
        found, id1, passed_any, last_ok, direct_chain = False, -1, False, None, 0
        for t, q, tl in direct:
            last_ok = passes(q)
            if not last_ok:
                continue
            passed_any = True
            ci = len(cand)
            cand.append((s, t, sim[q]))
            tl_idx = emit(tl, s)
            ok, c = attempt(s, t, "direct", 0)
            direct_chain = max(direct_chain, c)
            if not ok:
                hits["tlink_skipped"] += sum(passes(q2) for _, q2 in tl)
                continue
            if id1 < 0:
                id1 = local_id(s)
            A.append((id1, local_id(t), sim[q])); acc.append(ci)
            found = True
            links(s, id1, tl, tl_idx, "tlink", c)
        src_idx = emit(src_links, s) if passed_any else []
        if not found:
            if passed_any:
                hits["slink_gated"] += sum(passes(q2) for _, q2 in src_links)
            continue
        if last_ok is False and any(passes(q2) for _, q2 in src_links):
            hits["slink_after_failed"] += 1
        links(s, id1, src_links, src_idx, "slink", direct_chain)

    n = len(A)
    ei, ej, ew = np.empty(2 * n, np.int32), np.empty(2 * n, np.int32), np.empty(2 * n, np.float64)
    if n:
        a = np.array([x[0] for x in A], np.int32); b = np.array([x[1] for x in A], np.int32); w = np.array([x[2] for x in A])
        ei[0::2], ei[1::2], ej[0::2], ej[1::2], ew[0::2], ew[1::2] = a, b, b, a, w, w
    return Result(ei, ej, ew, l2g, cand, np.array(acc, np.int64), hits, chain, band, {qseg[q] for q in near})


# ------------------------------------------------------------------------------------------------------------ scenes
def pieces_scene(V, N, seed, neighbors, patterns, flip_every=0, tail_every=0):
    """synth.make_scene(collinear=True) in which view i sees every broken line (3D lines 2m, 2m+1: one infinite line with a gap)
    as patterns[i % len(patterns)]: None keeps the two pieces make_scene drew; otherwise a list of (t0, t1) fractions of the 2D
    segment from the start of piece 2m to the end of piece 2m+1, one segment each.  Pieces of different views overlap along the
    line wherever their fractions do, so collinear pieces of one view match each other's partners in another.
    flip_every > 0: every flip_every-th new piece has its end points swapped (its estimate points the other way: angles above 90
    degrees).  tail_every > 0: every tail_every-th line of a view with a pattern also gets a piece (1.05, 1.2) beyond its end,
    collinear with the line but seen by that view only (a collinear partner that gets no estimate)."""
    from line3dpp_b200 import synth
    sc = synth.make_scene(V, N, seed, neighbors, collinear=True)
    for i in range(V):
        pat = patterns[i % len(patterns)]
        if pat is None:
            continue
        ids, s = sc.line_ids[i], sc.segs[i]
        pos = {int(l): r for r, l in enumerate(ids)}
        out, lid, nnew = [], [], 0
        for r, l in enumerate(ids.tolist()):
            if l % 2 == 1 and l - 1 in pos:
                continue                                    # drawn with its even partner
            if l % 2 == 0 and l + 1 in pos:
                a, b = s[r, :2].astype(np.float64), s[pos[l + 1], 2:].astype(np.float64)
                pieces = list(pat) + ([(1.05, 1.2)] if tail_every and (l // 2) % tail_every == 0 else [])
                for t0, t1 in pieces:
                    p, q = a + t0 * (b - a), a + t1 * (b - a)
                    nnew += 1
                    if flip_every and nnew % flip_every == 0:
                        p, q = q, p
                    out.append(np.concatenate([p, q])); lid.append(l)
            else:
                out.append(s[r].astype(np.float64)); lid.append(l)
        perm = np.random.default_rng([seed, i, 1]).permutation(len(out))      # pieces of one line get unrelated segment ids
        sc.segs[i] = np.ascontiguousarray(np.array(out, np.float64)[perm].astype(np.float32)).reshape(-1, 4)
        sc.line_ids[i] = np.array(lid, np.int64)[perm]
    return sc


HALVES = [(0.0, 0.47), (0.53, 1.0)]
THIRDS = [(0.0, 0.3), (0.35, 0.65), (0.7, 1.0)]
OFFSET = [(0.12, 0.58), (0.64, 0.9)]

# name -> (V, N, seed, neighbours, patterns, flip_every, tail_every)
SCENES = {
    # every second view sees each broken line whole
    "whole_broken": (12, 500, 93, "ring3", [[(0.0, 1.0)], None], 0, 0),
    # halves, thirds and offset halves: pieces of different views overlap along the line, a view sees three pieces, partners
    # without an estimate and flipped pieces
    "overlap": (12, 400, 94, "ring3", [HALVES, THIRDS, None, OFFSET], 5, 4),
    # whole, thirds and offset halves on a denser neighbourhood
    "thirds": (10, 300, 95, "ring4", [[(0.0, 1.0)], THIRDS, OFFSET, THIRDS, HALVES], 3, 3),
}


def scene(name):
    V, N, seed, nb, pats, flip, tail = SCENES[name]
    return pieces_scene(V, N, seed, nb, pats, flip, tail)
