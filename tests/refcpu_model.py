"""A float64 restatement of the REF_CPU scoring sweep (use_GPU=false): scoringCPU (line3D.cc:1208-1294), similarityForScoring
(1417-1446), angleBetweenSeg3D (1571-1583) and filterMatches (1586-1669), with a bound on how far each build can be from it, and
the closure U of the decisions those bounds leave open.  numpy only; nothing here is the arithmetic under test.

Input: each view's scored list as the oracle returns it (OraclePipeline.scored: ids and depths, in list order), the scene's
cameras and each view's k (view_info).  The 3D geometry is the reference's double arithmetic, restated operation by operation
(the same IEEE double add / mul / div / sqrt in the same order, so P1, P2, dir, length and the target regularisers are those of
both builds bit for bit).  Every float operation of the reference is rounded to float32 where the reference rounds; the two libm
calls, acosf and expf, are evaluated in float64 and rounded once.  So the model differs from either build ONLY by the error of
that build's acosf / expf, carried through the float operations that follow them.

The in-band width.  With ulp(x) <= 2^-23 |x| for a normal float x:
  * acosf: CUDA's libdevice <= 2 ulp (CUDA C++ Programming Guide, "Mathematical Functions", single precision), glibc <= 1 ulp
    (libm-test-ulps); the model's correctly rounded value is within 0.5 ulp.  dA = (u_acos + 0.5) ulp(A).
  * degrees = (float)((double)A / pi * 180): dD = dA * 180 / pi + 1 ulp(D) (two inputs dA apart round at most 1 ulp further apart);
    the fold 180 - D for D > 90 is exact (Sterbenz).
  * (-D * D) / two_sigA_sqr: dX = ((2 D + dD) dD + ulp(D^2)) / two_sigA_sqr + ulp(X).
  * sim_a = expf(X): dS = S (e^dX - 1) + (u_exp + 0.5) ulp(S).
  * the depth terms expf(-e * e / reg): the argument is the same float in every build, dS = (u_exp + 0.5) ulp(S).
  * sim = min(sim_a, sim_p1, sim_p2): at most the largest of the three.
  A term whose inputs are bit-identical in every build and whose function value is exact (expf(0) = 1, acosf(1) = 0) has no
  error at all.  Near sim_t = 0.5 this is W ~ 2-9 ulps of 0.5 (1e-7 .. 3e-7 at sigma_a = 10 degrees); band_width() reports it.
  A similarity is IN BAND when |sim - 0.5| <= W of the GPU build (the wider one): there either build may decide sim > 0.5
  either way.  Everywhere else both builds decide as the model does.

Scores.  score3D is a float sum built with the reference's running per-camera maximum (add the first value of a camera, replace
it by a larger one: score -= best; score += sim).  Two builds whose similarities differ by at most W run the same operations
on inputs at most sum(W) apart, so their scores differ by at most E = the W of every similarity that enters plus 1 ulp of the
running sum for every operation on an input that can differ (a replacement whose two values lie within their W of each other
may go either way: both values' W and two operations are counted).  E = 0 means bit-identical in every build.  E is ~1e-6 of
the score on these scenes, tighter than the old rtol = 1e-5.

The closure U, in processing order (ascending camID, compute_matches):
  * an in-band similarity makes its entry's score uncertain: it lies in [lo, hi], the score with that similarity 0 and above 0.5;
  * an uncertain score whose sign can change (lo = 0 < hi) makes the inverse entry it activates uncertain (storeInverseMatches,
    line3D.cc:1672-1699, when the target view is processed later): if the oracle has that entry its similarities with the rest
    of the target segment's list become [0, s]; if not, the other build may have it, and every other entry of that list may
    gain up to 1 (one similarity <= 1 of a camera);
  * an uncertain entry that can be the view's maximum makes every filter decision of that view uncertain;
  * two matches of a segment into one view with bit-identical overlaps are listed in the reference's heap order, which the GPU
    matcher does not reproduce: the segment's list is compared with such runs sorted, and its scores get 2 ulps more per entry
    (the per-camera maximum is the same in either order, the float updates that build it are not);
  * a keep decision (score > 0 and score > 0.1 max) or best decision (the first largest kept score; best > 0.75) that the
    bounds cannot settle makes that segment's kept set and estimate uncertain.
"""
from __future__ import annotations

import dataclasses

import numpy as np

ULP = 2.0 ** -23                 # ulp(x) <= ULP * |x| for a normal float32 x
LIBM_ULPS = {"gpu": (2.0, 2.0), "cpu": (1.0, 1.0)}     # (acosf, expf): CUDA libdevice, glibc
MODEL_ULPS = 0.5                 # the model rounds a float64 libm value once
SIM_T = np.float32(0.5)          # L3D_DEF_MIN_SIMILARITY_3D
MIN_BEST = np.float32(0.75)      # L3D_DEF_MIN_BEST_SCORE_3D
PERC = np.float32(0.1)           # L3D_DEF_MIN_BEST_SCORE_PERC
EPS = 1e-12                      # L3D_EPS
PI_D = 3.14159265358979323846
f32 = np.float32


# ---------------------------------------------------------------------------------------------------------- geometry
def _inv3(a):
    """the cofactor inverse of the reference's 3x3 (oracle/l3d_oracle.cc inverse)"""
    c00 = a[1][1] * a[2][2] - a[1][2] * a[2][1]; c01 = a[1][2] * a[2][0] - a[1][0] * a[2][2]; c02 = a[1][0] * a[2][1] - a[1][1] * a[2][0]
    i = 1.0 / (a[0][0] * c00 + a[0][1] * c01 + a[0][2] * c02)
    return [[c00 * i, (a[0][2] * a[2][1] - a[0][1] * a[2][2]) * i, (a[0][1] * a[1][2] - a[0][2] * a[1][1]) * i],
            [c01 * i, (a[0][0] * a[2][2] - a[0][2] * a[2][0]) * i, (a[0][2] * a[1][0] - a[0][0] * a[1][2]) * i],
            [c02 * i, (a[0][1] * a[2][0] - a[0][0] * a[2][1]) * i, (a[0][0] * a[1][1] - a[0][1] * a[1][0]) * i]]


def _mul(a, b):
    """3x3 product, each element ((a0 b0 + a1 b1) + a2 b2)"""
    return [[a[i][0] * b[0][j] + a[i][1] * b[1][j] + a[i][2] * b[2][j] for j in range(3)] for i in range(3)]


class Cameras:
    """the views in the reference's working frame (Line3D::translate, line3D.cc:500-536: minus the per-axis median of the camera
    centres), double rays of every segment end point (View::getNormalizedRay) and each view's k"""

    def __init__(self, K, R, t, segs, k, cam_ids=None):
        V = len(K)
        self.cam_ids = [int(c) for c in (cam_ids if cam_ids is not None else range(V))]
        self.pos = {c: i for i, c in enumerate(self.cam_ids)}
        Rt = [[[float(R[v][j][i]) for j in range(3)] for i in range(3)] for v in range(V)]
        C = []
        for v in range(V):
            nt = [float(t[v][i]) * -1.0 for i in range(3)]
            C.append([Rt[v][i][0] * nt[0] + Rt[v][i][1] * nt[1] + Rt[v][i][2] * nt[2] for i in range(3)])
        tr = []
        for i in range(3):
            co = sorted(c[i] for c in C if abs(c[i]) > EPS)
            tr.append(co[len(co) // 2] if co else 0.0)
        self.C = np.array([[c[i] + tr[i] * -1.0 for i in range(3)] for c in C])
        self.k = np.array([float(x) for x in k], np.float32)
        self.rays = []
        for v in range(V):
            M = _mul(Rt[v], _inv3([[float(x) for x in row] for row in K[v]]))
            s = np.asarray(segs[v], np.float32).astype(np.float64)
            self.rays.append((self._ray(M, s[:, 0], s[:, 1]), self._ray(M, s[:, 2], s[:, 3])))

    @staticmethod
    def _ray(M, x, y):
        r = [M[i][0] * x + M[i][1] * y + M[i][2] * 1.0 for i in range(3)]
        n = np.sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2])
        return np.stack([r[0] / n, r[1] / n, r[2] / n], 1)

    @classmethod
    def of_scene(cls, sc, k):
        return cls(sc.K, sc.R, sc.t, sc.segs, k, sc.cam_ids)

    @classmethod
    def of_inputs(cls, inp, k):
        return cls(inp["K"], inp["R"], inp["t"], inp["segs"], k)

    def unproject(self, cam, seg, d1, d2):
        """View::unprojectSegment + Segment3D: P1, P2, dir (double) and the float length"""
        v = self.pos[cam]
        r1, r2 = self.rays[v][0][seg], self.rays[v][1][seg]
        C = self.C[v]
        P1 = C + r1 * d1.astype(np.float64)[:, None]
        P2 = C + r2 * d2.astype(np.float64)[:, None]
        a = P1 - P2
        length = np.sqrt(a[:, 0] * a[:, 0] + a[:, 1] * a[:, 1] + a[:, 2] * a[:, 2]).astype(np.float32)
        b = P2 - P1
        n = np.sqrt(b[:, 0] * b[:, 0] + b[:, 1] * b[:, 1] + b[:, 2] * b[:, 2])
        ok = length.astype(np.float64) > EPS
        d = np.where(ok[:, None], b / np.where(n > 0, n, 1.0)[:, None], 0.0)
        return P1, P2, d, np.where(ok, length, f32(0))

    def regularizer(self, cam, P):
        """View::regularizerFrom3Dpoint of view cam (view.cc:445-448)"""
        a = P - self.C[self.pos[cam]]
        return (np.sqrt(a[..., 0] * a[..., 0] + a[..., 1] * a[..., 1] + a[..., 2] * a[..., 2]) * float(self.k[self.pos[cam]])).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------- similarities
def _ulp(x):
    return ULP * np.abs(np.asarray(x, np.float64))


def _acosf(c):
    return np.arccos(c.astype(np.float64)).astype(np.float32)


def _expf(x):
    return np.exp(x.astype(np.float64)).astype(np.float32)


def sims(dot_p, e1, e2, reg1, reg2, two_sigA_sqr, zero):
    """similarityForScoring of pairs (arrays broadcast): dot_p the float dot of the two directions, e1 / e2 the float depth
    differences, reg1 / reg2 the own entry's regularisers, zero: a segment without length.  Returns (sim before truncation,
    {build: W})."""
    c = np.clip(dot_p, f32(-1), f32(1)).astype(np.float32)
    A = _acosf(c)
    raw = (A.astype(np.float64) / PI_D * 180.0).astype(np.float32)
    D = np.where(raw > f32(90), f32(180) - raw, raw).astype(np.float32)      # exact: raw in (90, 180]
    X = ((-D) * D).astype(np.float32) / f32(two_sigA_sqr)
    X = X.astype(np.float32)
    sa = _expf(X)
    x1 = (((-e1) * e1).astype(np.float32) / reg1).astype(np.float32)
    x2 = (((-e2) * e2).astype(np.float32) / reg2).astype(np.float32)
    s1, s2 = _expf(x1), _expf(x2)
    with np.errstate(invalid="ignore"):
        s = np.fmin(sa, np.fmin(s1, s2)).astype(np.float32)
    s = np.where(zero, f32(0), s)
    W = {}
    for b, (ua, ue) in LIBM_ULPS.items():
        dA = np.where(c == f32(1), 0.0, (ua + MODEL_ULPS) * _ulp(A))
        dD = np.where(dA > 0, dA * (180.0 / PI_D) * (1 + 1e-12) + _ulp(raw), 0.0)
        D64 = np.abs(D.astype(np.float64))
        dX = np.where(dD > 0, ((2 * D64 + dD) * dD + _ulp(D64 * D64)) / float(two_sigA_sqr) + _ulp(X), 0.0)
        ea = lambda x, S: np.where(x == 0, 0.0, (ue + MODEL_ULPS) * _ulp(S))
        wa = sa.astype(np.float64) * np.expm1(dX) + np.where((X == 0) & (dX == 0), 0.0, (ue + MODEL_ULPS) * _ulp(sa))
        with np.errstate(invalid="ignore"):
            w = np.fmax(wa, np.fmax(ea(x1, s1), ea(x2, s2)))
        W[b] = np.where(zero | np.isnan(s), 0.0, w)
    return s, W


# ---------------------------------------------------------------------------------------------------------- one view
@dataclasses.dataclass
class ViewResult:
    cam: int
    seg: np.ndarray                # src_seg of every entry (the scored list's order)
    score: np.ndarray              # the model's score3D (float64 holding the float32 value)
    E: dict                        # build -> per entry bound of |score_build - score|
    lo: np.ndarray                 # the score's interval: lo == hi == score unless the entry is uncertain
    hi: np.ndarray
    slack: np.ndarray              # what the builds may add around [lo, hi] (their E and the rounding of the sums)
    uncertain: np.ndarray          # entry in U: an in-band similarity or an uncertain partner in its list
    in_band: np.ndarray            # entry with an in-band similarity
    sim_gap: np.ndarray            # per entry: min over its similarities of |sim - 0.5| - W (<= 0: in band; inf: none)
    near: np.ndarray               # (entry, sim - 0.5, W) of every similarity within 1e-4 of 0.5
    vmax: float
    vmax_at: int                   # the entry attaining the view maximum (the first one)
    vmax_uncertain: bool
    lim: float                     # 0.1 * max in float
    perc_margin: np.ndarray        # per entry: score - lim
    best_at: dict                  # segment -> entry of its best kept match
    best_margin: dict              # segment -> best score - 0.75
    kept: np.ndarray               # the model's kept flags (score > 0, score > lim, and the segment's best > 0.75)
    kept_u: set                    # segments whose kept set or estimate is uncertain
    events: dict                   # how many segments each event brought into U: "sim", "order", "vmax", "perc", "best"
    ties: set                      # segments whose list holds a tie run (tie_runs): their order is compared sorted


def _pad_pow2(n):
    return 1 << max(0, int(n - 1).bit_length())


class _Entries:
    """the per-entry quantities of a view's list the similarities need"""

    def __init__(self, cams, cam, m):
        self.n = len(m)
        self.seg = m["src_seg"].astype(np.int64)
        self.tc = m["tgt_cam"].astype(np.int64)
        self.d1, self.d2 = m["d_p1"].astype(np.float32), m["d_p2"].astype(np.float32)
        P1, P2, self.dr, self.length = cams.unproject(cam, self.seg, self.d1, self.d2)
        k = cams.k[cams.pos[cam]]
        sig1, sig2 = self.d1 * k, self.d2 * k
        reg1, reg2 = (f32(2) * sig1) * sig1, (f32(2) * sig2) * sig2
        s1t, s2t = np.zeros(self.n, np.float32), np.zeros(self.n, np.float32)
        for t in np.unique(self.tc):
            w = self.tc == t
            s1t[w], s2t[w] = cams.regularizer(int(t), P1[w]), cams.regularizer(int(t), P2[w])
        self.reg1 = (f32(0.5) * (reg1 + (f32(2) * s1t) * s1t)).astype(np.float32)
        self.reg2 = (f32(0.5) * (reg2 + (f32(2) * s2t) * s2t)).astype(np.float32)


def _score_lists(x, idx, valid, gone_mask, two_sigA_sqr, out):
    """scoringCPU's loop for the own entries idx[g, i] (lists padded to one length, valid marks real positions) against every
    position j of their list, all lists of the chunk at once"""
    G, Lp = idx.shape
    I, J = idx[:, :, None], idx[:, None, :]
    dot = (x.dr[I, 0] * x.dr[J, 0] + x.dr[I, 1] * x.dr[J, 1] + x.dr[I, 2] * x.dr[J, 2]).astype(np.float32)
    zero = (x.length[I].astype(np.float64) < EPS) | (x.length[J].astype(np.float64) < EPS)
    s, W = sims(dot, x.d1[I] - x.d1[J], x.d2[I] - x.d2[J], x.reg1[I], x.reg2[I], two_sigA_sqr, zero)
    counts = valid[:, :, None] & valid[:, None, :] & (x.tc[I] != x.tc[J])
    gap = np.where(counts, np.abs(s.astype(np.float64) - 0.5) - W["gpu"], np.inf)
    gap = np.where(np.isnan(gap), np.inf, gap)
    inb = gap <= 0
    with np.errstate(invalid="ignore"):
        sv = np.where(counts & (s > SIM_T), s, f32(0)).astype(np.float32)
    # [lo, hi] of every similarity: in band, 0 or above 0.5; with a partner one build may lack, 0 or s
    s_lo = np.where(inb | gone_mask[J], 0.0, sv)
    s_hi = np.where(inb, np.maximum(s.astype(np.float64), 0.5) + W["gpu"], sv)
    u_pair = inb | (counts & gone_mask[J] & (sv > 0))
    # the running per-camera maximum, position by position
    cam_j = x.tc[idx]
    slot = np.argmax(cam_j[:, :, None] == cam_j[:, None, :], axis=2)      # first position of the same camera in the list
    sc = np.zeros((G, Lp), np.float32)
    Eb = {b: np.zeros((G, Lp)) for b in LIBM_ULPS}
    best = np.zeros((G, Lp, Lp), np.float32); seen = np.zeros((G, Lp, Lp), bool)
    wbest = {b: np.zeros((G, Lp, Lp)) for b in LIBM_ULPS}
    lo_c, hi_c = np.zeros((G, Lp, Lp)), np.zeros((G, Lp, Lp))
    gi, ii = np.meshgrid(np.arange(G), np.arange(Lp), indexing="ij")
    for j in range(Lp):
        act, sj = counts[:, :, j], sv[:, :, j]
        sl = np.broadcast_to(slot[:, j][:, None], (G, Lp))
        first = act & ~seen[gi, ii, sl]
        cur = best[gi, ii, sl]
        repl = act & ~first & (sj > cur)
        new = np.where(first, sc + sj, np.where(repl, (sc - cur) + sj, sc)).astype(np.float32)
        for b in LIBM_ULPS:
            wj, wc = np.where(sj > 0, W[b][:, :, j], 0.0), wbest[b][gi, ii, sl]
            near = act & ~first & ~repl & ((wj + wc) > 0) & (np.abs(sj.astype(np.float64) - cur) <= wj + wc)
            e_first = Eb[b] + wj
            e_first += np.where(e_first > 0, _ulp(np.abs(new) + e_first), 0.0)
            e_rep = Eb[b] + wj + wc
            e_rep += np.where(e_rep > 0, 2 * _ulp(np.abs(sc) + np.abs(new) + e_rep), 0.0)
            Eb[b] = np.where(first, e_first, np.where(repl | near, e_rep, Eb[b]))
            wbest[b][gi, ii, sl] = np.where(first | repl, wj, np.where(near, np.maximum(wj, wc), wc))
        best[gi, ii, sl] = np.where(first | repl, sj, cur)
        seen[gi, ii, sl] |= act
        lo_c[gi, ii, sl] = np.where(act, np.maximum(lo_c[gi, ii, sl], s_lo[:, :, j]), lo_c[gi, ii, sl])
        hi_c[gi, ii, sl] = np.where(act, np.maximum(hi_c[gi, ii, sl], s_hi[:, :, j]), hi_c[gi, ii, sl])
        sc = new
    own = idx[valid]
    out["score"][own] = sc[valid]
    for b in LIBM_ULPS:
        out["E"][b][own] = Eb[b][valid]
    # each camera's maximum counted once: the slots are the first positions of the cameras
    first_pos = (slot == np.arange(Lp)[None, :])[:, None, :]
    out["lo"][own] = (lo_c * first_pos).sum(2)[valid]
    out["hi"][own] = (hi_c * first_pos).sum(2)[valid]
    out["unc"][own] = u_pair.any(2)[valid]
    out["inb"][own] = inb.any(2)[valid]
    out["gap"][own] = gap.min(2)[valid]
    g, i, j = np.nonzero(np.abs(np.where(counts, s.astype(np.float64), np.inf) - 0.5) < 1e-4)
    if len(g):
        out["near"].append(np.stack([idx[g, i].astype(np.float64), s[g, i, j].astype(np.float64) - 0.5, W["gpu"][g, i, j]], 1))


CHUNK = 1 << 20                  # pairs evaluated at once


def score_view(cams, cam, m, two_sigA_sqr, gone=(), phantom=None):
    """scoringCPU + filterMatches of view cam's scored list m.  gone: indices of entries that one build may lack (their
    similarities are [0, s]); phantom: {segment: {camera}}: lists one build may hold an extra inverse entry in"""
    x = _Entries(cams, cam, m)
    n, seg = x.n, x.seg
    assert n == 0 or (np.diff(seg) >= 0).all(), "a scored list holds each segment's entries together, in segment order"
    gone_mask = np.zeros(n, bool)
    gone_mask[list(gone)] = True
    out = dict(score=np.zeros(n, np.float32), E={b: np.zeros(n) for b in LIBM_ULPS}, lo=np.zeros(n), hi=np.zeros(n),
               unc=np.zeros(n, bool), inb=np.zeros(n, bool), gap=np.full(n, np.inf), near=[])
    starts = np.flatnonzero(np.r_[True, seg[1:] != seg[:-1]]) if n else np.zeros(0, np.int64)
    ends = np.r_[starts[1:], n].astype(np.int64)
    lens = ends - starts
    pads = np.array([_pad_pow2(v) for v in lens.tolist()], np.int64)
    for Lp in sorted(set(pads.tolist())):
        grp = np.flatnonzero(pads == Lp)
        step = max(1, CHUNK // (Lp * Lp))
        for c0 in range(0, len(grp), step):
            g = grp[c0:c0 + step]
            idx = starts[g][:, None] + np.arange(Lp)[None, :]
            valid = idx < ends[g][:, None]
            _score_lists(x, np.where(valid, idx, starts[g][:, None]), valid, gone_mask, two_sigA_sqr, out)
    score, E, unc = out["score"], out["E"], out["unc"]
    lo, hi = out["lo"], out["hi"]
    for sg, pcs in (phantom or {}).items():      # every entry of another camera may gain up to 1 per extra entry
        w = (seg == sg) & ~np.isin(x.tc, list(pcs))
        hi[w] += len(pcs)
        unc[seg == sg] = True
    score64 = score.astype(np.float64)
    lo, hi = np.where(unc, lo, score64), np.where(unc, hi, score64)
    L = np.bincount(seg, minlength=int(seg.max()) + 1)[seg] if n else np.zeros(0)
    slack = E["gpu"] + E["cpu"] + 2 * L * _ulp(hi + 1.0)
    ev = {"sim": len(set(seg[out["inb"]].tolist()))}
    # matches of one segment into one view with bit-identical overlaps: the matcher's order among them is the reference's heap
    # order, which the GPU matcher does not reproduce.  The per-camera maximum is the same in either order, its float updates
    # are not: the segment's scores get 2 more ulps per list entry, its list order is compared with those runs sorted.
    tie = tie_runs(m)
    ties = set(seg[tie].tolist())
    for sg in ties:
        w = seg == sg
        unc[w] = True
        slack[w] += 2 * L[w] * _ulp(hi[w] + 1.0)
    ev["order"] = len(ties)

    # filterMatches: the view maximum, 10 % of it, each segment's best
    vmax = float(score.max()) if n else 0.0
    vmax_at = int(np.argmax(score)) if n else -1
    vm_cert = float(score64[~unc].max()) if (~unc).any() else 0.0
    Emax = float(E["gpu"].max() + E["cpu"].max()) if n else 0.0
    vmax_unc = bool(unc.any() and (hi[unc] + slack[unc]).max() >= vm_cert - Emax)
    lim = float(PERC * f32(vmax))
    dlim = 0.1 * Emax + (_ulp(lim) if Emax > 0 else 0.0)
    keep = (score > 0) & (score > f32(lim))
    margin = score64 - lim
    tol = E["gpu"] + E["cpu"] + dlim
    keep_u = np.where(unc, ((lo - slack <= lim + dlim) & (hi + slack > lim - dlim)) | ((lo <= 0) & (hi > 0)),
                      (np.abs(margin) <= tol) & (tol > 0))
    kept_u = set(np.unique(seg).tolist()) if vmax_unc else set()
    ev["vmax"] = len(kept_u)
    ev["perc"] = len(set(seg[keep_u].tolist()) - kept_u)
    kept_u |= set(seg[keep_u].tolist()) | set((phantom or {}).keys()) | set(seg[gone_mask].tolist())
    best_at, best_margin = {}, {}
    nb = 0
    T = E["gpu"] + E["cpu"]
    for a, b_ in zip(starts.tolist(), ends.tolist()):
        sg = int(seg[a])
        ks = [i for i in range(a, b_) if keep[i]]
        if not ks:
            continue
        bi = ks[0]
        for i in ks[1:]:
            if score[i] > score[bi]:
                bi = i
        best_at[sg], best_margin[sg] = bi, float(score64[bi]) - float(MIN_BEST)
        tie = any(i != bi and T[bi] + T[i] > 0 and abs(score64[i] - score64[bi]) <= T[bi] + T[i] for i in ks)
        if sg not in kept_u and (tie or (T[bi] > 0 and abs(best_margin[sg]) <= T[bi])):
            kept_u.add(sg)
            nb += 1
    ev["best"] = nb
    for sg in set(seg.tolist()) - {s_ for s_, m_ in best_margin.items() if m_ > 0}:
        keep[seg == sg] = False              # a segment whose best match is not above 0.75 keeps nothing
    near = np.concatenate(out["near"]) if out["near"] else np.zeros((0, 3))
    return ViewResult(cam, seg, score64, E, lo, hi, slack, unc, out["inb"], out["gap"], near, vmax, vmax_at, vmax_unc, lim, margin,
                      best_at, best_margin, keep, kept_u, ev, ties)


def _tie_key(m):
    return np.stack([m["src_seg"].astype(np.int64), m["tgt_cam"].astype(np.int64),
                     np.ascontiguousarray(m["overlap"]).view(np.uint32).astype(np.int64)], 1)


def tie_runs(m):
    """entries of m in a run of consecutive entries with one segment, one target view and bit-identical overlaps"""
    if len(m) < 2:
        return np.zeros(len(m), bool)
    k = _tie_key(m)
    same = (k[1:] == k[:-1]).all(1)
    return np.r_[same, False] | np.r_[False, same]


def canonical(m):
    """the permutation that sorts every tie run of m (tie_runs) by target segment and leaves everything else in place"""
    if len(m) < 2:
        return np.arange(len(m))
    k = _tie_key(m)
    run = np.cumsum(np.r_[True, ~(k[1:] == k[:-1]).all(1)])
    return np.lexsort((m["tgt_seg"], run))


# ---------------------------------------------------------------------------------------------------------- the whole sweep
@dataclasses.dataclass
class SweepResult:
    views: dict                    # cam -> ViewResult
    gone: dict                     # cam -> entries (indices into its scored list) one build may lack
    phantom: dict                  # cam -> {segment: {camera}}: an extra inverse entry one build may hold
    inverse_events: int

    def size(self):
        """|U|: segments whose list, scores, kept set or estimate the bounds leave open"""
        return sum(len(self.u_segments(c)) for c in self.views)

    def u_segments(self, cam):
        v = self.views[cam]
        return set(v.seg[v.uncertain].tolist()) | v.kept_u | set(self.phantom.get(cam, {})) | set(v.seg[list(self.gone.get(cam, ()))].tolist())

    def events(self):
        out = {"inverse": self.inverse_events}
        for v in self.views.values():
            for k, x in v.events.items():
                out[k] = out.get(k, 0) + x
        return out


def sweep(cams, scored, two_sigA_sqr):
    """the model over every view in processing order; scored: cam -> the oracle's scored list"""
    views, gone, phantom = {}, {}, {}
    order = sorted(scored)
    rank = {c: i for i, c in enumerate(order)}
    n_inv = 0
    for cam in order:
        m = scored[cam]
        r = score_view(cams, cam, m, two_sigA_sqr, gone.get(cam, ()), phantom.get(cam, {}))
        views[cam] = r
        sign_u = (r.lo <= 0) & (r.hi > 0)
        for i in np.flatnonzero(sign_u).tolist():
            t = int(m["tgt_cam"][i])
            if rank.get(t, -1) <= rank[cam]:
                continue                   # the target is processed: no inverse entry either way
            ts, ss = int(m["tgt_seg"][i]), int(m["src_seg"][i])
            mt = scored[t]
            hit = np.flatnonzero((mt["src_seg"] == ts) & (mt["tgt_cam"] == cam) & (mt["tgt_seg"] == ss))
            if len(hit):
                gone.setdefault(t, set()).update(hit.tolist())
            else:
                phantom.setdefault(t, {}).setdefault(ts, set()).add(cam)
            n_inv += 1
    return SweepResult(views, gone, phantom, n_inv)


def band_width(res):
    """the largest W (GPU build) of a similarity within 1e-4 of 0.5 over the sweep, 0 if there is none"""
    w = [float(v.near[:, 2].max()) for v in res.views.values() if len(v.near)]
    return max(w) if w else 0.0


# ---------------------------------------------------------------------------------------------------------- comparing two runs
IDS = ("src_seg", "tgt_cam", "tgt_seg")


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def check_run(res, scored_o, kept_o, est_o, scored_g, kept_g, est_g):
    """a REF_CPU run (scored_g / kept_g: cam -> list, est_g: (best, P)) against the oracle's (scored_o, kept_o, est_o) on which
    the model ran: outside U everything agrees (lists and order, depths bit for bit, score3D within E_gpu + E_cpu, kept sets,
    best matches, estimates bit for bit); inside U only what its event permits (the list without the uncertain entries, the score
    inside its interval).  Returns counts of what was compared."""
    st = dict(entries=0, exact=0, u_entries=0, kept=0, est=0)
    for cam, v in res.views.items():
        o, g = scored_o[cam], scored_g(cam)
        keep_o = np.ones(len(o), bool)
        keep_o[list(res.gone.get(cam, ()))] = False
        drop = {(int(o["src_seg"][i]), int(o["tgt_cam"][i]), int(o["tgt_seg"][i])) for i in res.gone.get(cam, ())}
        ph = res.phantom.get(cam, {})
        keep_g = np.array([(s, c, t) not in drop and c not in ph.get(s, ()) for s, c, t in zip(*(g[f].tolist() for f in IDS))], bool)
        io = np.flatnonzero(keep_o)
        oo, gg = o[keep_o], g[keep_g]
        po_, pg_ = canonical(oo), canonical(gg)
        oo, gg, io = oo[po_], gg[pg_], io[po_]
        assert not (po_ != np.arange(len(po_))).any() or v.ties, f"view {cam}: tie runs the model did not see"
        assert len(oo) == len(gg), f"view {cam}: {len(gg)} entries outside U, oracle {len(oo)}"
        for f in IDS:
            assert np.array_equal(gg[f], oo[f]), f"view {cam}: list order / membership differs in {f} outside U"
        for f in ("overlap", "d_p1", "d_p2", "d_q1", "d_q2"):
            assert np.array_equal(_bits(gg[f]), _bits(oo[f])), f"view {cam}: {f} not bit-identical"
        sg, so = gg["score3D"].astype(np.float64), oo["score3D"].astype(np.float64)
        E = (v.E["gpu"] + v.E["cpu"])[io]
        cert = ~v.uncertain[io]
        bad = cert & (np.abs(sg - so) > E)
        assert not bad.any(), f"view {cam}: score3D beyond the libm bound at entries {np.flatnonzero(bad)[:8]}: " \
                              f"{sg[bad][:4]} vs {so[bad][:4]}, bound {E[bad][:4]}"
        lo, hi = v.lo[io] - v.slack[io], v.hi[io] + v.slack[io]
        out = ~cert & ((sg < lo) | (sg > hi))
        assert not out.any(), f"view {cam}: uncertain scores outside their interval: {sg[out][:4]} not in {lo[out][:4]}, {hi[out][:4]}"
        st["entries"] += int(cert.sum()); st["exact"] += int((cert & (sg == so)).sum()); st["u_entries"] += int((~cert).sum())
        # kept sets of the segments U does not reach
        ku = np.array(sorted(v.kept_u), np.int64)
        ko, kg = kept_o[cam], kept_g(cam)
        ko, kg = ko[~np.isin(ko["src_seg"], ku)], kg[~np.isin(kg["src_seg"], ku)]
        ko, kg = ko[canonical(ko)], kg[canonical(kg)]
        assert len(ko) == len(kg), f"view {cam}: {len(kg)} kept matches outside U, oracle {len(ko)}"
        for f in IDS:
            assert np.array_equal(kg[f], ko[f]), f"view {cam}: kept matches differ in {f} outside U"
        st["kept"] += len(ko)
    # estimates
    (bo, po_), (bg, pg) = est_o, est_g
    uset = {(c, s) for c, v in res.views.items() for s in v.kept_u}
    ko = {(int(b["src_cam"]), int(b["src_seg"])): i for i, b in enumerate(bo)}
    kg = {(int(b["src_cam"]), int(b["src_seg"])): i for i, b in enumerate(bg)}
    assert set(ko) - uset == set(kg) - uset, "segments with an estimate differ outside U"
    for key in set(ko) - uset:
        a, b = bo[ko[key]], bg[kg[key]]
        assert (a["tgt_cam"], a["tgt_seg"]) == (b["tgt_cam"], b["tgt_seg"]), f"best match of {key}"
        assert np.array_equal(po_[ko[key]].view(np.uint64), pg[kg[key]].view(np.uint64)), f"estimate of {key} not bit-identical"
    st["est"] = len(set(ko) - uset)
    return st


def run_model(cams, pipe, cam_ids, two_sigA_sqr):
    """the model on an oracle pipeline that has run matchImages: (result, scored, kept, estimates)"""
    scored = {int(c): pipe.scored(c) for c in cam_ids}
    kept = {int(c): pipe.matches(c) for c in cam_ids}
    return sweep(cams, scored, two_sigA_sqr), scored, kept, pipe.estimates()


def kept_decisions(res):
    """segments whose kept set or estimate U reaches"""
    return sum(len(v.kept_u) for v in res.views.values())
