"""Hand-built match lists that put the scoring sweep's decisions (csrc/l3d_pipeline.cu) at their thresholds, with a float64 model
of where each case lies.  numpy only; nothing here is the arithmetic under test.

The lists replace what matching produced (Line3D::setShard's exchange on the product, orc_set_match_source on the oracle) and obey
what the matcher guarantees: at most kNN entries per row, distinct target segments below Nt, four positive depths, an overlap in
(epi_overlap, 1].  Every case owns its segments, so no case changes another one's lists:

  background   matches of the segments of one ground-truth 3D line (views 0-6), depths where the rays pass the line: the
               reconstruction has something to cluster
  orientation  one record whose depths put checkMatchOrientation's cosine (line3D.cc:811-858) in a named band, on a direct entry
               (the source's list) or on an inverse entry (the target's list, checked when the target is processed; a second
               record to a third view with the same source depths makes the source score it > 0, so that the inverse entry exists)
  similarity   two records of one segment to two views whose depth difference or angle puts K_score_matches' similarity at the
               sim_t truncation or at the sweep's shortcuts (q_thr, cos_thr)
  filter       segments whose two best scores tie, scores on both sides of 0.75 and of 0.1 * the view's maximum; view 7 only
               receives single inverse entries, so none of its scores is positive

Bands of the orientation cosine c = ray_mid . dir (T1 = cos((double)0.098174771f), T2 = cos((double)3.043417886f); the reference
keeps a match iff T2 < c < T1):
  fast_*        |c| more than 1e-4 from 0.99518473f: the float fast path decides
  dbl_*         inside the float margin, more than 1e-9 from the threshold: the double shortcut decides
  acos_*        within 1e-9 of the threshold (and at least 1e-10 away): acos decides
  bug_*         (T2, -0.99518472667 - 1e-9): the double shortcut with the symmetric constant dropped these
  short_*       3D direction just below / above 1 % of the depths (|d|^2 against 1e-4 (d1^2 + d2^2))
  zero          depths of 1e-12: the 3D segment has no length (n^2 <= 1e-20, P1 == P2 in float: NaN direction)
"""
from __future__ import annotations

import dataclasses
import math

import numpy as np

from line3dpp_b200 import synth

REC_DT = np.dtype([("tgt_seg", "<u4"), ("overlap", "<f4"), ("d_p1", "<f4"), ("d_p2", "<f4"), ("d_q1", "<f4"), ("d_q2", "<f4")])

T1 = math.cos(float(np.float32(0.098174771)))            # 0.99518472640441780
T2 = math.cos(float(np.float32(3.043417886)))            # -0.99518473132192450
C0F = float(np.float32(0.99518473))                      # the float fast path's threshold
OLD_C2 = -0.99518472667                                  # the symmetric constant the double shortcut used for T2
SIM_T = 0.5                                              # L3D_DEF_MIN_SIMILARITY_3D
KNN = 10
V, NSEG, SEED = 8, 300, 11
NB = 120                                                 # segments below this index carry the background
D0 = 4.0                                                 # depth of the hand-built records

# name: (lo, hi) of the signed cosine; p_* lie at the pi/32 threshold, m_* and bug_* at the 31 pi/32 one
ORIENT_BANDS = {
    "p_fast_keep": (C0F - 1e-4 - 6e-5, C0F - 1e-4 - 3e-5), "p_fast_drop": (C0F + 1e-4 + 3e-5, C0F + 1e-4 + 6e-5),
    "p_dbl_keep": (T1 - 7e-5, T1 - 2e-9), "p_dbl_drop": (T1 + 2e-9, T1 + 7e-5),
    "p_acos_keep": (T1 - 9e-10, T1 - 1e-10), "p_acos_drop": (T1 + 1e-10, T1 + 9e-10),
    "m_fast_keep": (-C0F + 1e-4 + 3e-5, -C0F + 1e-4 + 6e-5), "m_fast_drop": (-C0F - 1e-4 - 6e-5, -C0F - 1e-4 - 3e-5),
    "m_dbl_keep": (T2 + 5e-9, T2 + 7e-5), "m_dbl_drop": (T2 - 7e-5, T2 - 2e-9),
    "m_acos_drop": (T2 - 9e-10, T2 - 1e-10),
    "bug_acos_keep": (T2 + 1e-10, T2 + 9e-10), "bug_dbl_keep": (T2 + 1.1e-9, OLD_C2 - 1e-9 - 1e-10),
}
SHORT_BANDS = {"short_below": (0.8e-4, 0.97e-4), "short_above": (1.03e-4, 1.2e-4)}
# cases placed in every orientation band, on direct entries and on inverse entries each
ORIENT_WANT = 3

# parameter sets of match_images: sigma_a 10 (default), 1, 75 (cos_thr live at ~88.7 deg), 76 (cos_thr off from 89 deg), and a
# fixed regulariser (k = 0.2 / 4 for every view: depth differences up to ~7 % of the depth stay similar, so angles at the cos_thr
# shortcut are reachable with depth terms near 1)
PARAMS = {"sa10": dict(sigma_a=10.0), "sa1": dict(sigma_a=1.0), "sa75": dict(sigma_a=75.0), "sa76": dict(sigma_a=76.0),
          "fixed": dict(sigma_a=10.0, sigma_p=-0.2, const_reg_depth=4.0)}


def scene():
    """8 views, every view the neighbour of every other (28 pairs), 300 segments each"""
    return synth.make_scene(V, NSEG, SEED, "dense")


def f32(x):
    return np.float32(x)


def _inv3(a):
    """the cofactor inverse the reference's Eigen 3x3 uses"""
    c00 = a[1, 1] * a[2, 2] - a[1, 2] * a[2, 1]; c01 = a[1, 2] * a[2, 0] - a[1, 0] * a[2, 2]; c02 = a[1, 0] * a[2, 1] - a[1, 1] * a[2, 0]
    det = a[0, 0] * c00 + a[0, 1] * c01 + a[0, 2] * c02
    i = 1.0 / det
    return np.array([[c00 * i, (a[0, 2] * a[2, 1] - a[0, 1] * a[2, 2]) * i, (a[0, 1] * a[1, 2] - a[0, 2] * a[1, 1]) * i],
                     [c01 * i, (a[0, 0] * a[2, 2] - a[0, 2] * a[2, 0]) * i, (a[0, 2] * a[1, 0] - a[0, 0] * a[1, 2]) * i],
                     [c02 * i, (a[0, 1] * a[2, 0] - a[0, 0] * a[2, 1]) * i, (a[0, 0] * a[1, 1] - a[0, 1] * a[1, 0]) * i]])


def _unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


class Geometry:
    """double rays (View::getNormalizedRay), camera centres and regularisers k of a scene under one parameter set"""

    def __init__(self, sc, params):
        self.sc = sc
        self.RtKinv = [sc.R[v].T @ _inv3(sc.K[v]) for v in range(sc.num_views)]
        self.C = np.array([-sc.R[v].T @ sc.t[v] for v in range(sc.num_views)])
        self.r1, self.r2, self.rm = [], [], []
        for v in range(sc.num_views):
            s = sc.segs[v].astype(np.float64)
            h = lambda x, y: _unit(np.stack([x, y, np.ones_like(x)], 1) @ self.RtKinv[v].T)
            self.r1.append(h(s[:, 0], s[:, 1])); self.r2.append(h(s[:, 2], s[:, 3]))
            self.rm.append(h(0.5 * (s[:, 0] + s[:, 2]), 0.5 * (s[:, 1] + s[:, 3])))
        sigma_p = params.get("sigma_p", 2.5)
        if sigma_p < 0:
            self.k = [float(f32(abs(sigma_p)) / f32(params["const_reg_depth"]))] * sc.num_views
        else:
            self.k = []
            for v in range(sc.num_views):       # View::specificSpatialReg (view.cc:307-314)
                pp = np.array([sc.K[v][0, 2], sc.K[v][1, 2], 1.0])
                a = _unit(self.RtKinv[v] @ pp) @ _unit(self.RtKinv[v] @ (pp + np.array([f32(max(0.1, sigma_p)), 0, 0])))
                self.k.append(float(f32(math.sin(math.acos(min(max(a, -1.0), 1.0))))))
        sa = min(abs(params.get("sigma_a", 10.0)), 90.0)
        self.angle_reg = float(f32(2.0) * f32(sa) * f32(sa))
        self.q_thr = float(f32(1.01) * f32(-math.log(SIM_T)))
        ang = math.sqrt(self.q_thr * self.angle_reg)
        self.cos_thr = float(f32(math.cos(ang * math.pi / 180.0) * (1.0 - 1e-4))) if ang < 89.0 else -1.0

    def cosine(self, v, s, d1, d2):
        """ray_mid . dir of the match (view v, segment s, depths d1, d2) in double; arrays broadcast"""
        d1, d2 = np.asarray(d1, np.float64)[..., None], np.asarray(d2, np.float64)[..., None]
        d = self.r2[v][s] * d2 - self.r1[v][s] * d1
        return (d @ self.rm[v][s]) / np.linalg.norm(d, axis=-1)

    def short_ratio(self, v, s, d1, d2):
        d1, d2 = np.asarray(d1, np.float64), np.asarray(d2, np.float64)
        d = self.r2[v][s] * d2[..., None] - self.r1[v][s] * d1[..., None]
        return (d * d).sum(-1) / (d1 * d1 + d2 * d2)

    def direction(self, v, s, d1, d2):
        return _unit(self.r2[v][s] * float(d2) - self.r1[v][s] * float(d1))

    def pos_reg(self, v, s, d1, d2, tgt):
        """K_score_matches' pos_reg1, pos_reg2 of an entry of view v's segment s (depths d1, d2) matched into view tgt"""
        out = []
        for r, d in ((self.r1[v][s], d1), (self.r2[v][s], d2)):
            P = self.C[v] + r * float(d)
            reg_t = float(f32(np.linalg.norm(P - self.C[tgt]) * self.k[tgt]))
            sig = float(f32(self.k[v]) * f32(d))
            out.append(0.5 * (2 * sig * sig + 2 * reg_t * reg_t))
        return out

    def sim(self, v, s, own, other, own_tgt):
        """similarity of entry `own` (d1, d2) with entry `other` of the same segment list (float64 model of K_score_matches)"""
        pr = self.pos_reg(v, s, own[0], own[1], own_tgt)
        e = [float(f32(own[i]) - f32(other[i])) for i in range(2)]
        dp = float(self.direction(v, s, *own) @ self.direction(v, s, *other))
        ang = math.degrees(math.acos(min(max(dp, -1.0), 1.0)))
        ang = 180.0 - ang if ang > 90.0 else ang
        return min(math.exp(-ang * ang / self.angle_reg), math.exp(-e[0] ** 2 / pr[0]), math.exp(-e[1] ** 2 / pr[1]))


def orientation_keeps(c):
    """checkMatchOrientation's decision from the double cosine: pi/32 < acos(c) < 31 pi/32 with the float thresholds"""
    a = np.arccos(np.clip(c, -1.0, 1.0))
    return (a > float(np.float32(0.098174771))) & (a < float(np.float32(3.043417886)))


def ulps(x, n):
    """the 2n+1 floats around float32(x)"""
    x = np.float32(x)
    out = [x]
    lo = hi = x
    for _ in range(n):
        lo = np.nextafter(lo, np.float32(-np.inf)); hi = np.nextafter(hi, np.float32(np.inf))
        out += [lo, hi]
    return np.sort(np.array(out, np.float32))


@dataclasses.dataclass
class Case:
    kind: str            # orientation | similarity | filter
    band: str
    view: int            # the view whose list holds the decided entry
    seg: int
    tgt_cam: int         # the entry's other view
    tgt_seg: int
    expect: object       # orientation: kept (bool); similarity: score > 0 (bool); filter: see build()
    inverse: bool = False
    info: dict = dataclasses.field(default_factory=dict)


class Lists:
    """match lists of every view pair, rows of records, and the cases placed in them"""

    def __init__(self, sc, geo):
        self.sc, self.geo = sc, geo
        self.pairs = [tuple(int(x) for x in p) for p in synth.view_pairs(sc.neighbors, sc.cam_ids)]
        self.rows = {p: [[] for _ in range(len(sc.segs[p[0]]))] for p in self.pairs}
        self.free = [list(range(NB, len(sc.segs[v]))) for v in range(sc.num_views)]
        self.cases: list[Case] = []
        self.rng = np.random.default_rng(SEED)

    def take(self, v, pred=None):
        for i, s in enumerate(self.free[v]):
            if pred is None or pred(s):
                return self.free[v].pop(i)
        return None

    def add(self, src, s, tgt, t, dp, dq, overlap=0.75):
        row = self.rows[(src, tgt)][s]
        assert len(row) < KNN and all(r[0] != t for r in row) and min(*dp, *dq) > 0
        row.append((t, overlap, float(f32(dp[0])), float(f32(dp[1])), float(f32(dq[0])), float(f32(dq[1]))))

    # ---- the records as the product's match buffers and as the oracle's match source
    def buffers(self):
        """counts int32[rows] and records REC_DT[rows, KNN] of all pairs in pair order (the layout of l3d_match_device_buffers)"""
        rows = [r for p in self.pairs for r in self.rows[p]]
        counts = np.array([len(r) for r in rows], np.int32)
        recs = np.zeros((len(rows), KNN), REC_DT)
        for i, r in enumerate(rows):
            for j, x in enumerate(r):
                recs[i, j] = x
        return counts, recs

    def source(self, match_dt):
        def fn(src, tgt, Ns, Nt, knn, cap):
            counts = np.zeros(Ns, np.int32)
            out = np.zeros((Ns, cap), match_dt)
            for r, row in enumerate(self.rows[(src, tgt)]):
                counts[r] = len(row)
                for j, (t, ov, a, b, c, d) in enumerate(row):
                    assert t < Nt
                    out[r, j] = (src, r, tgt, t, ov, 0.0, a, b, c, d)
            return counts, out
        return fn


def _ray_depth(C, r, P, dL):
    """depth along the ray C + lambda r of its closest approach to the line P + mu dL"""
    w = C - P
    a, b, c, d, e = r @ r, r @ dL, dL @ dL, r @ w, dL @ w
    return (b * e - c * d) / (a * c - b * b)


def _background(L):
    sc, g = L.sc, L.geo
    for (u, v) in L.pairs:
        if v == V - 1:
            continue                    # view 7 gets no background: its lists stay without positive scores
        ids_v = {}
        for t in range(NB):
            ids_v.setdefault(int(sc.line_ids[v][t]), t)
        for s in range(NB):
            t = ids_v.get(int(sc.line_ids[u][s]))
            if t is None:
                continue
            ln = sc.lines3d[int(sc.line_ids[u][s])]
            P, dL = ln[:3], ln[3:] - ln[:3]
            dp = [_ray_depth(g.C[u], g.r1[u][s], P, dL), _ray_depth(g.C[u], g.r2[u][s], P, dL)]
            dq = [_ray_depth(g.C[v], g.r1[v][t], P, dL), _ray_depth(g.C[v], g.r2[v][t], P, dL)]
            if min(dp + dq) > 0.1:
                L.add(u, s, v, t, dp, dq, overlap=0.9)


def _solve_d2(f, d1, target, lo=1e-4, hi=1e4):
    """d2 with f(d2) = target for an f increasing in d2 on [lo * d1, hi * d1], or None"""
    a, b = lo * d1, hi * d1
    if not (f(a) < target < f(b)):
        return None
    for _ in range(200):
        m = math.sqrt(a * b)
        if f(m) < target:
            a = m
        else:
            b = m
    return 0.5 * (a + b)


def place_cosine(g, v, s, lo, hi, d1=D0):
    """float depths (d1, d2) near d1 whose double cosine lies in (lo, hi), from a scan of adjacent floats, or None"""
    mid = 0.5 * (lo + hi)
    d2 = _solve_d2(lambda x: float(g.cosine(v, s, d1, x)), d1, mid)
    if d2 is None:
        return None
    for n in (8, 64):
        A, B = np.meshgrid(ulps(d1, n), ulps(d2, n), indexing="ij")
        c = g.cosine(v, s, A.ravel(), B.ravel())
        ok = np.flatnonzero((c > lo) & (c < hi))
        if len(ok):
            i = ok[np.argmin(np.abs(c[ok] - mid))]
            return float(A.ravel()[i]), float(B.ravel()[i]), float(c[i])
    return None


def place_short(g, v, s, lo, hi, d1=D0):
    mid = 0.5 * (lo + hi)
    base = g.short_ratio(v, s, d1, d1)
    if not base < lo:
        return None
    d2 = d1
    step = d1 * 1e-3
    while g.short_ratio(v, s, d1, d2) < mid and d2 < 2 * d1:
        d2 += step
    a, b = d2 - step, d2
    for _ in range(100):
        m = 0.5 * (a + b)
        if g.short_ratio(v, s, d1, m) < mid:
            a = m
        else:
            b = m
    d2 = float(f32(b))
    r = float(g.short_ratio(v, s, d1, d2))
    return (d1, d2, float(g.cosine(v, s, d1, d2))) if lo < r < hi else None


def _orientation_cases(L):
    sc, g = L.sc, L.geo
    nice = (D0, D0)
    seg_len = [np.hypot(sc.segs[v][:, 2] - sc.segs[v][:, 0], sc.segs[v][:, 3] - sc.segs[v][:, 1]) for v in range(V)]
    bands = [(b, "cos", lo, hi) for b, (lo, hi) in ORIENT_BANDS.items()] + [(b, "short", lo, hi) for b, (lo, hi) in SHORT_BANDS.items()] + \
        [("zero", "zero", 0, 0)]
    k = 0
    for band, how, lo, hi in bands:
        for inverse in (False, True):
            for rep in range(ORIENT_WANT):
                for _attempt in range(40):
                    k += 1
                    # direct: decided on u's segment s; inverse: on v's segment t (v processed after u)
                    u = k % 5 if inverse else k % 7
                    v = u + 1 + (k // 7) % (V - 1 - u)
                    w = next((x for x in range(u + 1, V) if x != v), None)
                    host = v if inverse else u
                    pred = (lambda x, h=host: seg_len[h][x] < 40) if how == "short" else None
                    hs = L.take(host, pred)
                    if hs is None:
                        break
                    d1 = D0 * (1.0 + 0.01 * rep)
                    if how == "cos":
                        got = place_cosine(g, host, hs, lo, hi, d1)
                    elif how == "short":
                        got = place_short(g, host, hs, lo, hi, d1)
                    else:
                        got = (1e-12, 1e-12, 0.0)
                    if got is None:
                        if how != "short":          # a short segment that misses its band is not used again
                            L.free[host].insert(0, hs)
                        continue
                    a, b, c = got
                    keep = True if how == "zero" else bool(orientation_keeps(c))
                    if inverse:
                        s = L.take(u); ws = L.take(w)
                        L.add(u, s, v, hs, nice, (a, b)); L.add(u, s, w, ws, nice, nice)
                        L.cases.append(Case("orientation", band, v, hs, u, s, keep, True, dict(c=c, d=(a, b))))
                    else:
                        t = L.take(v)
                        L.add(u, hs, v, t, (a, b), nice)
                        L.cases.append(Case("orientation", band, u, hs, v, t, keep, False, dict(c=c, d=(a, b))))
                    break


def _sim_pair(L, u, band, ratio, kind, want_keep):
    """segment s of view u with X -> v1 at (D0, D0) and Y -> v2: kind 'depth' shifts both depths by delta (same direction), 'angle'
    by +delta / -delta (a rotation); ratio = the largest depth term's e^2 / (pos_reg ln(1/sim_t)), or the angle's
    angle^2 / (angle_reg ln(1/sim_t))"""
    g = L.geo
    v1, v2 = u + 1, u + 2
    s = L.take(u)
    X = (D0, D0)
    ln = -math.log(SIM_T)
    if kind == "depth":
        pr = g.pos_reg(u, s, *X, v1)
        delta = math.sqrt(ratio * ln * min(pr))
        Y = (float(f32(D0 + delta)), float(f32(D0 + delta)))
        e = [float(f32(X[i]) - f32(Y[i])) for i in range(2)]
        got = max(e[i] * e[i] / pr[i] for i in range(2)) / ln
        term = int(np.argmax([e[i] * e[i] / pr[i] for i in range(2)]))
    else:
        target = math.sqrt(ratio * ln * g.angle_reg)
        def ang(dl):
            dp = float(g.direction(u, s, *X) @ g.direction(u, s, D0 + dl, D0 - dl))
            return math.degrees(math.acos(min(max(dp, -1.0), 1.0)))
        a, b = 0.0, 0.9 * D0
        if ang(b) < target:
            L.free[u].insert(0, s)
            return None
        for _ in range(100):
            m = 0.5 * (a + b)
            a, b = (m, b) if ang(m) < target else (a, m)
        Y = (float(f32(D0 + b)), float(f32(D0 - b)))
        pr = g.pos_reg(u, s, *X, v1)
        e = [float(f32(X[i]) - f32(Y[i])) for i in range(2)]
        if max(e[i] * e[i] / pr[i] for i in range(2)) > 0.5 * ln:      # the depth terms must stay well above sim_t
            L.free[u].insert(0, s)
            return None
        dp = float(g.direction(u, s, *X) @ g.direction(u, s, *Y))
        got = math.degrees(math.acos(min(dp, 1.0))) ** 2 / g.angle_reg / ln
        term = dp
    t1, t2 = L.take(v1), L.take(v2)
    L.add(u, s, v1, t1, X, (D0, D0)); L.add(u, s, v2, t2, Y, (D0, D0))
    c = Case("similarity", band, u, s, v1, t1, want_keep, info=dict(ratio=got, term=term, Y=Y, sim=g.sim(u, s, X, Y, v1)))
    L.cases.append(c)
    return c


SIM_BANDS = {"q_in": (0.995, True), "q_full": (1.005, False), "q_short": (1.015, False)}
ANG_BANDS = {"a_in": (0.993, True), "a_full": (1.003, False), "a_short": (1.04, False)}


def _similarity_cases(L):
    g = L.geo
    for band, (ratio, keep) in SIM_BANDS.items():
        for i in range(6):
            _sim_pair(L, i % 5, band, ratio, "depth", keep)
    for band, (ratio, keep) in ANG_BANDS.items():
        for i in range(6):
            c = _sim_pair(L, i % 5, band, ratio, "angle", keep)
            if c is None:
                continue
            dp = c.info["term"]
            # which side of the cos_thr shortcut the pair lies on (the float cosine is good to ~1e-7)
            c.info["shortcut"] = g.cos_thr > 0 and abs(dp) < g.cos_thr * (1 - 1e-5)
            if g.cos_thr > 0 and abs(abs(dp) - g.cos_thr) < 1e-5 * g.cos_thr:
                L.cases.remove(c)


def _filter_cases(L):
    g = L.geo
    # view 0: one segment matched into all 7 other views at the same depths: every entry scores the same ~6 (a tie of 7), the
    # view's maximum, so 0.1 * max ~ 0.6
    s = L.take(0)
    ts = []
    for v in range(1, V):
        t = L.take(v); ts.append(t)
        L.add(0, s, v, t, (D0, D0), (D0, D0))
    L.cases.append(Case("filter", "tie", 0, s, 1, ts[0], 7))
    # ties of two: X -> u+1, Y -> u+2 at the same depths
    for u in range(1, 6):
        s = L.take(u)
        t1, t2 = L.take(u + 1), L.take(u + 2)
        L.add(u, s, u + 1, t1, (D0, D0), (D0, D0)); L.add(u, s, u + 2, t2, (D0, D0), (D0, D0))
        L.cases.append(Case("filter", "tie", u, s, u + 1, t1, 2))
    ln = math.log

    def shift_for(u, s, own, tgt, sim):
        pr = min(g.pos_reg(u, s, own, own, tgt))
        return math.sqrt(pr * -ln(sim))
    # best score just below / above 0.75 (X and Y similar to each other at ~0.745 / ~0.755 both ways)
    for u in range(0, 6):
        for band, sim in (("best_below_075", 0.742), ("best_above_075", 0.758)):
            s = L.take(u)
            v1, v2 = (u + 1, u + 2)
            dl = shift_for(u, s, D0, v1, sim)
            Y = (float(f32(D0 + dl)),) * 2
            sx, sy = g.sim(u, s, (D0, D0), Y, v1), g.sim(u, s, Y, (D0, D0), v2)
            if (band == "best_below_075") != (max(sx, sy) < 0.75) or abs(max(sx, sy) - 0.75) < 2e-3:
                continue
            t1, t2 = L.take(v1), L.take(v2)
            L.add(u, s, v1, t1, (D0, D0), (D0, D0)); L.add(u, s, v2, t2, Y, (D0, D0))
            L.cases.append(Case("filter", band, u, s, v1, t1, band == "best_above_075", info=dict(sx=sx, sy=sy)))
    # view 0: A1 -> 1 at D0, A2 -> 2 at D0 + x (similar to A1), A3 -> 3 at D0 - y, similar to A1 only, scoring ~0.55 or ~0.65
    # against the view's 0.1 * max ~ 0.6; A1's score (~1.5) makes the segment's best > 0.75
    for band, sim in (("perc_below", 0.55), ("perc_above", 0.65)) * 3:
        s = L.take(0)
        y = shift_for(0, s, D0, 3, sim)
        x = 0.4 * y
        A1, A2, A3 = (D0, D0), (float(f32(D0 + x)),) * 2, (float(f32(D0 - y)),) * 2
        s31, s32 = g.sim(0, s, A3, A1, 3), g.sim(0, s, A3, A2, 3)
        s1 = g.sim(0, s, A1, A2, 1) + g.sim(0, s, A1, A3, 1)
        if s32 > 0.45 or s1 < 0.8 or abs(s31 - 0.6) < 0.03:
            continue
        t = [L.take(v) for v in (1, 2, 3)]
        L.add(0, s, 1, t[0], A1, (D0, D0)); L.add(0, s, 2, t[1], A2, (D0, D0)); L.add(0, s, 3, t[2], A3, (D0, D0))
        L.cases.append(Case("filter", band, 0, s, 3, t[2], band == "perc_above", info=dict(score=s31)))


def build(sc, params):
    """the lists of scene sc under parameter set params (a dict of match_images arguments) and their cases"""
    L = Lists(sc, Geometry(sc, params))
    _background(L)
    _orientation_cases(L)
    _similarity_cases(L)
    _filter_cases(L)
    return L


# ---------------------------------------------------------------------------------------------------------- outcomes
def band_counts(L, kind=None):
    out = {}
    for c in L.cases:
        if kind is None or c.kind == kind:
            key = (c.band, c.inverse) if c.kind == "orientation" else c.band
            out[key] = out.get(key, 0) + 1
    return out


def has_entry(scored, c):
    """does the scored list of c.view hold c's entry"""
    m = scored
    return bool(np.any((m["src_seg"] == c.seg) & (m["tgt_cam"] == c.tgt_cam) & (m["tgt_seg"] == c.tgt_seg)))


def entry(scored, c):
    m = scored
    i = np.flatnonzero((m["src_seg"] == c.seg) & (m["tgt_cam"] == c.tgt_cam) & (m["tgt_seg"] == c.tgt_seg))
    return m[i[0]] if len(i) else None


def check_cases(L, scored, kept, estimates):
    """the outcome of every case in a run's results (scored / kept: per view id; estimates: best records); returns the list of
    (band, case) that disagree with the model"""
    bad = []
    est = {(int(b["src_cam"]), int(b["src_seg"])): b for b in estimates}
    for c in L.cases:
        sc_, kp = scored[c.view], kept[c.view]
        if c.kind == "orientation":
            if has_entry(sc_, c) != c.expect:
                bad.append((c.band + (" inverse" if c.inverse else " direct"), c))
        elif c.kind == "similarity":
            e = entry(sc_, c)
            if e is None or (float(e["score3D"]) > 0) != c.expect:
                bad.append((c.band, c))
        elif c.band == "tie":
            b = est.get((c.view, c.seg))
            seg = sc_[sc_["src_seg"] == c.seg]
            if b is None or len(seg) < c.expect or len(set(seg["score3D"].view(np.uint32).tolist())) != 1 \
                    or (int(b["tgt_cam"]), int(b["tgt_seg"])) != (int(seg[0]["tgt_cam"]), int(seg[0]["tgt_seg"])):
                bad.append((c.band, c))
        elif c.band.startswith("best_"):
            if ((c.view, c.seg) in est) != c.expect:
                bad.append((c.band, c))
        elif c.band.startswith("perc_"):
            if has_entry(kp, c) != c.expect or (c.view, c.seg) not in est:
                bad.append((c.band, c))
    return bad
