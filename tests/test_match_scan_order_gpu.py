"""The order in which k_match_topk scans a row's window pieces (l3d_match.cu scan_row: the arc class nearest the row's own span first,
then outward, the targets without an arc last) decides only when candidates reach the exact path, never which are kept.  On a scene
built to reach every ordering case - rows of span class 0 and of the last class, windows that wrap around 2^32 (two pieces of one
class), targets without an arc, source points at the epipole (rows that skip level 1), and views that take two passes over the ring -
the keep-all rows, whose order does not depend on the scan, must be the CPU oracle's, and the top-k rows for kNN 1, 10, 32 and 40 must
be the k best of the keep-all rows by (overlap descending, then the smaller target index), the order of the kernel's keys, so exact
ties in the k-th place are checked too.  Both semantics."""
import numpy as np
import pytest

from line3dpp_b200 import synth
from tests import level1_model as l1
from tests import util

PAIRS = np.array([(0, 1), (1, 0)], np.int32)
EPI = 0.25
KNNS = [1, 10, 32, 40]
RES = 6 * 512                       # target segments resident in one pass (MK_STAGES x MK_TT)


def _epipole(F):
    """the point of the source image whose epipolar line is zero: F e = 0"""
    e = np.linalg.svd(np.asarray(F, np.float64).reshape(3, 3))[2][-1]
    return e[:2] / e[2]


def _scene():
    sc = util.two_view_scene("forward", 3300, 41)                 # epipole inside both images: the pencil covers every direction
    rng = np.random.default_rng(7)
    for v, (s, t) in enumerate(PAIRS):
        ex, ey = _epipole(util.pair_F(sc, [(s, t)])[0])          # epipole of view v as the source of pair (v, 1 - v)
        extra = []
        for a in np.linspace(0.0, np.pi, 40, endpoint=False):
            c, d = np.cos(a), np.sin(a)
            extra += [(ex, ey, ex + 220 * c, ey + 220 * d),       # source point at the epipole: the row skips level 1
                      (ex - 250 * c, ey - 250 * d, ex + 250 * c, ey + 250 * d),            # through the epipole: no arc as a target
                      (ex + 400 * c, ey + 400 * d, ex + 700 * c, ey + 700 * d)]            # on one pencil line: span class 0
        for _ in range(120):                                      # long segments close to the epipole: spans of the last class
            x, y, a = ex + rng.uniform(-300, 300), ey + rng.uniform(-300, 300), rng.uniform(0, np.pi)
            extra.append((x - 600 * np.cos(a), y - 600 * np.sin(a), x + 600 * np.cos(a), y + 600 * np.sin(a)))
        extra = np.array(extra, np.float32)
        extra[:, 0::2] = np.clip(extra[:, 0::2], 0, synth.WIDTH - 1)
        extra[:, 1::2] = np.clip(extra[:, 1::2], 0, synth.HEIGHT - 1)
        sc.segs[v] = np.ascontiguousarray(np.concatenate([sc.segs[v], extra]))
    return sc


@pytest.fixture(scope="module")
def scene():
    return _scene()


def test_scene_reaches_every_scan_order_case(scene):
    """the rows and targets of pair (0, 1) reach each case of the piece order (l3d_match.cu scan_row), by the numpy restatement of
    the level-1 tables"""
    F = util.pair_F(scene, PAIRS[:1])[0]
    u, v, _ = l1.basis(F)
    ext = 1.0 / EPI + 0.5
    no_arc = sum(l1.target_arc(u, v, q, ext) is None for q in scene.segs[1])
    span_cls, wraps, skips = [], 0, 0
    for s in scene.segs[0]:
        k1, off1 = l1.line_kappa(u, v, l1.epipolar_line(F, s[0], s[1]))
        k2, off2 = l1.line_kappa(u, v, l1.epipolar_line(F, s[2], s[3]))
        if off1 or off2:
            skips += 1
            continue
        fwd = ((k2 - k1) & l1.M32) < 0x80000000
        ka, kb = (k1, k2) if fwd else (k2, k1)
        span_cls.append(min(l1.arc_class((kb - ka) & l1.M32), l1.NCLS - 1))
        wraps += ka < (1 << (l1.CLS0 + l1.NCLS - 1))             # the window of the last class wraps around 2^32
    span_cls = np.array(span_cls)
    assert len(scene.segs[1]) > RES and len(scene.segs[0]) > RES   # both directions take two passes
    assert skips >= 20 and no_arc >= 20 and wraps >= 20
    assert (span_cls == 0).sum() >= 20 and (span_cls == l1.NCLS - 1).sum() >= 20
    assert len(np.unique(span_cls)) == l1.NCLS


def _expected(oracle, scene, f64):
    """per pair: the oracle's keep-all rows (ascending target), as lists of records"""
    Fd = np.stack([synth.fundamental(scene.K[s], scene.R[s], scene.t[s], scene.K[t], scene.R[t], scene.t[t]).reshape(9) for s, t in PAIRS])
    RtKinv, C = synth.camera_blocks(scene)
    out = []
    for p, (s, t) in enumerate(PAIRS):
        cap = 512
        while True:
            if f64:
                oc, oo, _, _ = oracle.match_lines(oracle.lib().orc_match_lines_f64, scene.segs[s], scene.segs[t], Fd[p], RtKinv[s].reshape(9),
                                                  RtKinv[t].reshape(9), C[s], C[t], s, t, EPI, 0, f64=True, cap=cap)
            else:
                pi = util.pair_inputs(scene, s, t)
                oc, oo, _, _ = oracle.match_lines(oracle.lib().orc_match_lines_f32, pi["ls"], pi["lt"], pi["F"], pi["Rs"], pi["Rt"], pi["Cs"],
                                                  pi["Ct"], s, t, EPI, 0, cap=cap)
            if oc.max() <= cap:
                break
            cap = int(oc.max())
        out.append((oc, oo))
    return Fd, out


FIELDS = ("tgt_seg", "overlap", "d_p1", "d_p2", "d_q1", "d_q2")
ORACLE_FIELDS = {False: ("tgt_seg", "overlap"), True: FIELDS}


def _row(recs, n, fields):
    return [tuple(int(np.float32(e[f]).view(np.uint32)) if recs.dtype[f].kind == "f" else int(e[f]) for f in fields) for e in recs[:n]]


def _through_epipole(scene, s, t):
    """rows of pair (s, t) whose source segment's line passes within 2 px of its epipole.  For these F*p is rounding noise, and the
    oracle's restatement of the float kernel is known to keep a match that the reference's CUDA kernel drops (DESIGN.md section 9)"""
    ex, ey = _epipole(util.pair_F(scene, [(s, t)])[0])
    q = scene.segs[s].astype(np.float64)
    dx, dy = q[:, 2] - q[:, 0], q[:, 3] - q[:, 1]
    return np.abs(dx * (ey - q[:, 1]) - dy * (ex - q[:, 0])) / np.hypot(dx, dy) < 2.0


def _run(gpu_ctx, scene, Fd, f64, knn):
    if f64:
        gpu_ctx.match_pairs_f64(PAIRS, Fd, EPI, knn)
    else:
        gpu_ctx.match_pairs(PAIRS, util.pair_F(scene, PAIRS), EPI, knn if knn > 0 else -1)
    return [tuple(a.copy() for a in gpu_ctx.pair_matches(p, len(scene.segs[s]))) for p, (s, _) in enumerate(PAIRS)]


def _best(row, k):
    """the k best records of a keep-all row: overlap descending, then the smaller target index (the order of the kernel's keys)"""
    return row[np.lexsort((row["tgt_seg"], -row["overlap"].astype(np.float64)))][:k]


@pytest.mark.gpu
@pytest.mark.parametrize("f64", [False, True], ids=["ref_gpu", "ref_cpu"])
def test_scan_order_keeps_the_oracles_matches(gpu_ctx, oracle, scene, f64):
    """keep-all rows (ascending target) against the oracle; kNN 1, 10, 32 and 40 (best first) against the k best of the keep-all rows,
    every field bit for bit.  In float semantics the rows through their own epipole are compared with the keep-all rows only."""
    gpu_ctx.set_views(util.scene_descs(scene), scene.segs)
    Fd, want = _expected(oracle, scene, f64)
    every = _run(gpu_ctx, scene, Fd, f64, 0)
    for p, (s, t) in enumerate(PAIRS):
        (oc, oo), (counts, recs) = want[p], every[p]
        rows = np.arange(len(counts))
        if not f64:
            skip = _through_epipole(scene, s, t)
            assert 80 <= skip.sum() <= 200, skip.sum()
            rows = rows[~skip]
        bad = [int(r) for r in rows if counts[r] != oc[r] or _row(recs[r], counts[r], ORACLE_FIELDS[f64]) != _row(oo[r], oc[r], ORACLE_FIELDS[f64])]
        assert not bad, (f64, s, t, len(bad), [(r, int(counts[r]), int(oc[r])) for r in bad[:10]])
        assert counts.sum() > 20000
    for knn in KNNS:
        got = _run(gpu_ctx, scene, Fd, f64, knn)
        for p, (s, t) in enumerate(PAIRS):
            (ac, ar), (counts, recs) = every[p], got[p]
            bad = [r for r in range(len(counts)) if _row(recs[r], counts[r], FIELDS) != _row(_best(ar[r, :ac[r]], knn), min(ac[r], knn), FIELDS)]
            assert not bad, (f64, knn, s, t, len(bad), [(r, int(counts[r]), int(ac[r])) for r in bad[:10]])
