"""Rows of thousands of matches for the matcher's three per-row decisions (csrc/l3d_match.cu): the top-k key lists of k_match_topk /
k_match_cand, the count and store passes of keep-all (kNN <= 0), and k_sort_rows, which puts keep-all rows in target order and cuts
kNN > 32 rows to their k best.  numpy only; which target matches which row is decided by the CPU oracle, never by this file.

The rig is a rectified pair: every source view sits at (-0.3, 0, -4), every target view at (0.3, 0, -4), same K, no rotation, so the
epipolar lines are the image rows y = const and the float and double F have exact zeros off the (y, 1) block.  A source row is a
vertical segment of BAND px at x = XS; its epipolar band is the strip of image rows it spans.  Its matches are vertical target segments
that cover the strip, x = XS - disparity (depth about 4): the overlap is BAND / length, and the arithmetic of both semantics gives
the same float for two targets of the same length whose strip lies inside them, wherever they sit on the row or along the column:
  distinct    targets of distinct lengths (overlaps distinct values in (0.3, 0.96))
  tie         exact duplicates of one target (overlap and depths equal)
  tie_at_k    `prefix` distinct overlaps above (0.6 .. 0.96), then a run of targets of one length (overlap 0.5) shifted along the
              column, so their arcs of the epipolar pencil differ; the run's indices go to its ends in column order (smallest index at
              one end, the next at the other, ...), so that a tied winner sits where the scan meets it last, whichever way it runs
Rows sit PITCH px apart: no target reaches another row's strip.  Pads (vertical segments below every strip) make a target view as long
as asked without adding matches.  Each job is checked with the oracle under both semantics (orc_match_lines_f32: REF_GPU,
orc_match_lines_f64: REF_CPU), keep-all with `cap` = the longest wanted row: candidates that do not match, or do not give the run its
common overlap, are dropped, and the job is rebuilt until every row's count is the one asked for."""
from __future__ import annotations

import dataclasses

import numpy as np

from line3dpp_b200 import synth
from tests import util

EPI = 0.25
KNNS = (1, 2, 16, 17, 31, 32, 33, 100, 2000, 0, -1)
TOPK = tuple(k for k in KNNS if k > 0)
LENGTHS = tuple(sorted({n for k in TOPK for n in (k - 1, k, k + 1)} | {0, 1, 32, 33, 64, 200}))
# k_sort_rows (l3d_capi.cu run_keep_all): 24-byte records, SORT_SMEM_MAX = 200 KiB of shared memory per block, 4, 2 or 1 warps
REC_BYTES, SORT_SMEM_MAX = 24, 200 * 1024
ROW_LIMIT = SORT_SMEM_MAX // REC_BYTES                                    # 8533
SORT_BANDS = {2133: 4, 2134: 2, 4266: 2, 4267: 1, 8533: 1}               # longest row -> warps per block
GRID_BLOCKS_PER_SM = 16                                                   # k_sort_rows' grid: at most num_sms * 16 blocks

BAND = 20.0                                     # px: height of a source row's strip
XS = 2000.0                                     # px: column of the source rows
PITCH, Y0 = 120.0, 60.0                         # px between strips (targets reach < 47 px beyond theirs), first strip
ROWS_PER_VIEW = 17
PAD_Y = 2200.0                                  # pads: below every strip
Q = 1.0 / 256.0                                 # coordinate grid: lengths and shifts are exact in float


@dataclasses.dataclass
class Row:
    kind: str                   # "distinct", "tie", "tie_at_k", or "pad" (a row of the padding pair)
    n: int                      # matches wanted
    prefix: int = 0             # tie_at_k: distinct overlaps above the run


@dataclasses.dataclass
class Job:
    scene: synth.Scene
    pairs: np.ndarray           # (P, 2) int32
    rows: list                  # per pair: the Rows of its source view
    keep_all: dict              # semantics ("gpu" / "cpu") -> per pair (counts int32[Ns], records MATCH_DT[Ns, cap]) of the oracle
    runs: dict                  # (pair, row) -> target indices of the row's tie run in column order (tie_at_k rows)

    @property
    def longest(self) -> int:
        return max((max((r.n for r in rows), default=0) for rows in self.rows), default=0)

    def F32(self):
        return util.pair_F(self.scene, self.pairs)

    def F64(self):
        sc = self.scene
        return np.stack([synth.fundamental(sc.K[s], sc.R[s], sc.t[s], sc.K[t], sc.R[t], sc.t[t]).reshape(9) for s, t in self.pairs])


def _vseg(x, y1, length):
    return (x, y1, x, y1 + length)


def _q(v):
    return np.round(np.asarray(v, np.float64) / Q) * Q


def _candidates(rng, ya, row, extra):
    """candidate targets of one row (more than it needs): list of (segment, role), role "d" distinct, "t" tie-run / duplicate"""
    out = []
    x = lambda: XS - _q(rng.uniform(330.0, 420.0))

    def distinct(count, lo, hi):
        L = rng.choice(np.arange(np.ceil(BAND / hi / Q), np.floor(BAND / lo / Q)) * Q, size=count, replace=False)
        for l in L:
            off = _q(rng.uniform(0.2, l - BAND - 0.2))
            out.append((_vseg(x(), ya - off, l), "d"))

    if row.kind == "distinct":
        distinct(row.n + extra, 0.3, 0.96)
    elif row.kind == "tie":
        l = _q(rng.uniform(BAND / 0.9, BAND / 0.4))
        s = _vseg(x(), ya - _q((l - BAND) / 2), l)
        out += [(s, "t")] * row.n
    elif row.kind == "tie_at_k":
        distinct(row.prefix + extra, 0.6, 0.96)
        m = row.n - row.prefix
        l = 2.0 * BAND                          # overlap 0.5, below every distinct one
        offs = rng.choice(np.arange(1, int((l - BAND - 0.5) / Q)) * Q + 0.25, size=m + extra, replace=False)
        out += [(_vseg(x(), ya - off, l), "t") for off in offs]
    return out


def _oracle(scene, pairs, sem, caps):
    """keep-all rows of every pair under one semantics, caps[p] records per row of pair p"""
    from oracle import pyoracle as O
    out = []
    RtKinv, C = synth.camera_blocks(scene)
    for (s, t), cap in zip(pairs, caps):
        if sem == "gpu":
            pi = util.pair_inputs(scene, s, t)
            r = O.match_lines(O.lib().orc_match_lines_f32, pi["ls"], pi["lt"], pi["F"], pi["Rs"], pi["Rt"], pi["Cs"], pi["Ct"], s, t, EPI, 0,
                              cap=cap)
        else:
            F = synth.fundamental(scene.K[s], scene.R[s], scene.t[s], scene.K[t], scene.R[t], scene.t[t]).reshape(9)
            r = O.match_lines(O.lib().orc_match_lines_f64, scene.segs[s], scene.segs[t], F, RtKinv[s].reshape(9), RtKinv[t].reshape(9),
                              C[s], C[t], s, t, EPI, 0, f64=True, cap=cap)
        out.append((r[0], r[1]))
    return out


def _scene(src_segs, tgt_segs):
    """views 2j (source pose) and 2j+1 (target pose) hold the segments of pair j"""
    V = 2 * len(src_segs)
    K = np.array([[synth.FOCAL, 0, synth.WIDTH / 2.0], [0, synth.FOCAL, synth.HEIGHT / 2.0], [0, 0, 1.0]])
    t = np.array([[0.3, 0.0, 4.0] if v % 2 == 0 else [-0.3, 0.0, 4.0] for v in range(V)])     # t = -C
    segs = [None] * V
    segs[0::2], segs[1::2] = src_segs, tgt_segs
    segs = [np.ascontiguousarray(np.asarray(s, np.float64).reshape(-1, 4).astype(np.float32)) for s in segs]
    return synth.Scene(cam_ids=np.arange(V, dtype=np.uint32), K=np.repeat(K[None], V, 0), R=np.repeat(np.eye(3)[None], V, 0), t=t,
                       median_depth=np.full(V, 4.0, np.float32), segs=segs, neighbors=[np.zeros(0, np.uint32) for _ in range(V)])


def _pads(rng, n, y=PAD_Y):
    return [_vseg(_q(rng.uniform(10.0, synth.WIDTH - 10.0)), y + _q(rng.uniform(0.0, 60.0)), 20.0) for _ in range(n)]


def build(row_lists, seed, pad_targets=0, pad_rows=0, extra=None):
    """One pair per entry of row_lists (at most ROWS_PER_VIEW rows each); pad_rows > 0 puts a padding pair of that many source rows
    and one target first (rows that match nothing, before every crowded row); pad_targets pads every crowded target view."""
    rng = np.random.default_rng(seed)
    extra = extra if extra is not None else (lambda r: 8 + r.n // 10)
    src, pools = [], []
    for rows in row_lists:
        assert len(rows) <= ROWS_PER_VIEW
        src.append([_vseg(XS, Y0 + i * PITCH, BAND) for i in range(len(rows))])
        pools.append([_candidates(rng, Y0 + i * PITCH, r, extra(r)) for i, r in enumerate(rows)])
    # first pass: every candidate, in row order; which of them match (and at what overlap) is the oracle's word
    tgt = [[c[0] for pool in pp for c in pool] for pp in pools]
    caps = [max([1] + [len(pool) for pool in pp]) for pp in pools]
    first = {sem: _oracle(_scene(src, tgt), np.array([(2 * j, 2 * j + 1) for j in range(len(src))], np.int32), sem, caps)
             for sem in ("gpu", "cpu")}
    keep = []
    for j, rows in enumerate(row_lists):
        base, kept = 0, []
        for i, (r, pool) in enumerate(zip(rows, pools[j])):
            ov = {}
            for sem in ("gpu", "cpu"):
                cnt, recs = first[sem][j]
                ov[sem] = {int(e["tgt_seg"]) - base: float(e["overlap"]) for e in recs[i, :cnt[i]]}
            ok = [c for c in range(len(pool)) if c in ov["gpu"] and c in ov["cpu"]]
            d = [c for c in ok if pool[c][1] == "d"]
            t = [c for c in ok if pool[c][1] == "t"]
            if r.kind == "tie_at_k" and t:       # the run: the candidates that share its most common overlap under both semantics
                vals = [(ov["gpu"][c], ov["cpu"][c]) for c in t]
                common = max(set(vals), key=vals.count)
                t = [c for c, v in zip(t, vals) if v == common]
            want_d = r.n if r.kind == "distinct" else r.prefix if r.kind == "tie_at_k" else 0
            want_t = r.n - want_d
            assert len(d) >= want_d and len(t) >= want_t, ("too few matching candidates", j, i, r, len(d), len(t))
            kept.append([pool[c] for c in d[:want_d] + t[:want_t]])
            base += len(pool)
        keep.append(kept)
    # the job: targets in a random order, each tie run's indices put at the ends of the run in column order, pads mixed in
    tgt, runs = [], {}
    for j, kept in enumerate(keep):
        items = [(np.array(s, np.float64), i, role) for i, row in enumerate(kept) for s, role in row]
        items += [(np.array(s, np.float64), -1, "p") for s in _pads(rng, pad_targets)]
        idx = rng.permutation(len(items))
        segs = np.zeros((len(items), 4))
        for i in range(len(kept)):
            if row_lists[j][i].kind != "tie_at_k":
                continue
            run = [m for m, it in enumerate(items) if it[1] == i and it[2] == "t"]
            if not run:
                continue
            run.sort(key=lambda m: items[m][0][1])                        # column order
            slots = sorted(idx[m] for m in run)
            ends = [run[-1 - q // 2] if q % 2 == 0 else run[q // 2] for q in range(len(run))]
            for m, sl in zip(ends, slots):
                idx[m] = sl
            runs[(j, i)] = [int(idx[m]) for m in run]
        for m, it in enumerate(items):
            segs[idx[m]] = it[0]
        tgt.append(segs)
    pairs = [(2 * j, 2 * j + 1) for j in range(len(src))]
    rows = [list(r) for r in row_lists]
    if pad_rows > 0:                             # source rows strictly above every strip's reach, one target in the pad band
        src = [[_vseg(_q(rng.uniform(10.0, synth.WIDTH - 10.0)), 2.0, 10.0) for _ in range(pad_rows)]] + src
        tgt = [np.array(_pads(rng, 1))] + tgt
        pairs = [(2 * j, 2 * j + 1) for j in range(len(src))]
        rows = [[Row("pad", 0)] * pad_rows] + rows
        runs = {(j + 1, i): v for (j, i), v in runs.items()}
    scene = _scene(src, tgt)
    pairs = np.array(pairs, np.int32)
    caps = [max([1] + [r.n for r in rr]) for rr in rows]      # the longest wanted row of each pair: memory stays small
    job = Job(scene, pairs, rows, {sem: _oracle(scene, pairs, sem, caps) for sem in ("gpu", "cpu")}, runs)
    for sem in ("gpu", "cpu"):
        for p, rr in enumerate(rows):
            counts = job.keep_all[sem][p][0]
            assert counts.tolist() == [r.n for r in rr], ("the oracle's counts are not the ones asked for", sem, p)
    return job


# ------------------------------------------------------------------------------------------------ the jobs of the tests
def knn_rows():
    """every length of LENGTHS in every kind (tie_at_k: half distinct, then the run), and for every kNN of TOPK a row with k - 1
    distinct overlaps and a run of 4 across the k-th place"""
    rows = [Row("distinct", n) for n in LENGTHS] + [Row("tie", n) for n in LENGTHS]
    rows += [Row("tie_at_k", n, n // 2) for n in LENGTHS]
    rows += [Row("tie_at_k", k + 3, k - 1) for k in TOPK]
    rows.sort(key=lambda r: -r.n)               # spread the long rows over the pairs
    per = [[] for _ in range((len(rows) + ROWS_PER_VIEW - 1) // ROWS_PER_VIEW)]
    for i, r in enumerate(rows):
        per[i % len(per)].append(r)
    return per


def knn_job(seed=101):
    return build(knn_rows(), seed)


def band_job(longest, pad_rows, seed=202):
    """one crowded pair whose longest row is `longest` (with an all-tie row and a tie_at_k row beside it), after a padding pair of
    pad_rows rows"""
    rows = [Row("distinct", longest), Row("tie", 150), Row("tie_at_k", 120, 40)]
    return build([rows], seed + longest, pad_rows=pad_rows, pad_targets=500)


# ------------------------------------------------------------------------------------------------ the rows every kNN must give
def expected_rows(counts, recs, knn):
    """from keep-all rows: kNN > 0 the rows sorted by (overlap descending, tgt_seg ascending) and cut to kNN (counts clipped), kNN <= 0
    the rows in ascending tgt_seg.  Returns (counts, list of per-row record arrays)"""
    out_c, out_r = np.zeros(len(counts), np.int32), []
    for r in range(len(counts)):
        e = recs[r, :counts[r]]
        order = np.argsort(e["tgt_seg"], kind="stable") if knn <= 0 else np.lexsort((e["tgt_seg"], -e["overlap"].astype(np.float64)))[:knn]
        out_r.append(e[order])
        out_c[r] = len(order)
    return out_c, out_r


def tie_at(recs_sorted, k):
    """True when the k-th and (k+1)-th best of a row (sorted best first) have the same overlap: a tie run straddles the k-th place"""
    return len(recs_sorted) > k and recs_sorted["overlap"][k - 1] == recs_sorted["overlap"][k]


def sort_warps(stride):
    """warps per block of k_sort_rows at a keep-all stride, 0 where the call fails"""
    for w in (4, 2, 1):
        if REC_BYTES * stride * w <= SORT_SMEM_MAX:
            return w
    return 0
