"""l3d_affinity_matrix and l3d_affinity_edges against the float64 sequential restatement of computingAffinityMatrix
(tests/affinity_model.py), fed with what the context exports after the scoring sweep: the kept matches (l3d_get_view_matches), the
estimates (l3d_get_estimates) and the collinear lists (l3d_get_collinear).  The model orders the estimates by camID itself.

The contexts are driven through the C ABI so that k, median_depth, the sweep's thresholds and the affinity parameters are the test's:
the scenes of tests/affinity_model.py with the links off, at 2 px and at 5 px, under min_affinity 0.2 / 0.5 / 0.9, two_sigA_sqr
20 / 200 and med_scene_depth_lines 0 / the median / half the median (min_affinity moved by at most 3e-4 where a similarity lies
within 1e-5 of it: Run.settle); the "thirds" scene once more with filterMatches at 30 % of the
best score, where target links are rejected by earlier direct edges (see tests/test_affinity_model_cpu.py); REF_CPU matching, whose
kept lists are in append order; views handed over in shuffled camID order; views with 0 and 1 segments and without estimates;
nothing passing; links on with every list empty; a problem with more than 1e5 candidates; and the context's cache of the result."""
import ctypes as C
import functools

import numpy as np
import pytest

from line3dpp_b200 import synth
from tests import affinity_model as am
from tests import util

pytestmark = pytest.mark.gpu

RTOL = 1e-5                       # float32 device against the float64 model
COLLIN = (-1.0, 2.0, 5.0)
PARAMS = [(tsa, medf, ma) for ma in (0.2, 0.5, 0.9) for tsa in (20.0, 200.0) for medf in (0.0, 1.0, 0.5)]   # medf: x the median
DEFAULT = (200.0, 1.0, 0.5)
WORST = {"gap": 0.0, "chain": 0}  # the largest weight gap and the longest dependency chain seen, printed by test_report


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def median_depths(V):
    """per-view median depths around the scene's depth of 4 (some depths above, some below every cutoff)"""
    return (3.0 + 0.4 * (np.arange(V) % 5)).astype(np.float32)


class Run:
    """a context with a scene matched and scored; views handed to l3d_set_views in `order` (indices into the scene)"""

    def __init__(self, sc, order=None, f64=False, perc=0.1):
        from line3dpp_b200 import capi
        V = sc.num_views
        self.sc, self.order = sc, np.arange(V) if order is None else np.asarray(order)
        RtKinv, Cw = synth.camera_blocks(sc)
        self.k = np.array([2.5 / sc.K[v][0, 0] for v in range(V)], np.float32)
        self.md = median_depths(V)
        o = self.order
        self.nseg = [len(sc.segs[v]) for v in o]
        self.seg_off = np.concatenate([[0], np.cumsum(self.nseg)]).astype(np.int64)
        self.pos = {int(sc.cam_ids[v]): i for i, v in enumerate(o)}          # camID -> index in the l3d_set_views array
        self.descs = lambda md: capi.make_view_descs(sc.cam_ids[o], [sc.width] * V, [sc.height] * V, self.nseg, RtKinv[o], Cw[o], Cw[o],
                                                      self.k[o], md[o])
        ctx = self.ctx = capi.Context(0)
        L = ctx.L
        ctx.set_views(self.descs(self.md), [sc.segs[v] for v in o])
        pairs = synth.view_pairs(sc.neighbors, sc.cam_ids)                       # camIDs == scene indices
        idx = np.array([[self.pos[int(s)], self.pos[int(t)]] for s, t in pairs], np.int32).reshape(-1, 2)
        if f64:
            ctx.match_pairs_f64(idx, [synth.fundamental(sc.K[s], sc.R[s], sc.t[s], sc.K[t], sc.R[t], sc.t[t]) for s, t in pairs])
        else:
            ctx.match_pairs(idx, util.pair_F(sc, pairs))
        assert L.l3d_score_sweep(ctx.h, C.c_float(200.0), C.c_float(.5), C.c_float(.75), C.c_float(perc)) == 0
        self.collin = None

    def g(self, seg):
        """global segment index of (camID, segment)"""
        return int(self.seg_off[self.pos[seg[0]]] + seg[1])

    def links(self, dist_t):
        self.ctx.find_collinear(dist_t, 0)
        self.collin = dist_t

    def problem(self):
        """the model's input from the context's exports"""
        from line3dpp_b200 import capi
        ctx, L = self.ctx, self.ctx.L
        lists = []
        for i in range(len(self.order)):
            n = ctx._chk(L.l3d_get_view_matches(ctx.h, i, 1, None, C.c_longlong(0)), "l3d_get_view_matches")
            m = np.zeros(n, capi.MATCH_DT)
            if n:
                assert L.l3d_get_view_matches(ctx.h, i, 1, _p(m), C.c_longlong(n)) == n
            lists.append(m)
        n = ctx._chk(L.l3d_get_estimates(ctx.h, None, None, C.c_longlong(0)), "l3d_get_estimates")
        best, P = np.zeros(n, capi.MATCH_DT), np.zeros((n, 6), np.float64)
        if n:
            assert L.l3d_get_estimates(ctx.h, _p(best), _p(P), C.c_longlong(n)) == n
        col = None
        if self.collin is not None and self.collin > am.EPS:
            col = {int(self.sc.cam_ids[v]): ctx.collinear(i, self.nseg[i]) for i, v in enumerate(self.order)}
        views = {int(self.sc.cam_ids[v]): (np.float32(self.k[v]), np.float32(self.md[v])) for v in self.order}
        return am.problem(best, P, lists, col, views)

    def median(self):
        return float(np.median(self.md))

    def args(self, tsa, medf, ma):
        return (self.ctx.h, C.c_float(tsa), C.c_float(medf * self.median()), C.c_float(ma))

    def model_args(self, tsa, medf, ma):
        return float(np.float32(tsa)), float(np.float32(medf * self.median())), float(np.float32(ma))

    def model(self, pr, tsa, medf, ma):
        return am.restate(pr, *self.model_args(tsa, medf, ma))

    def settle(self, pr, tsa, medf, ma):
        """(params, model result) with min_affinity moved by the least multiple of 1e-4 that leaves no similarity within the model's
        guard band of it, so that float32 rounding cannot flip a decision"""
        for d in (0.0, 1e-4, -1e-4, 2e-4, -2e-4, 3e-4, -3e-4):
            r = self.model(pr, tsa, medf, ma + d)
            if r.band == 0:
                return (tsa, medf, ma + d), r
        raise AssertionError(f"no min_affinity near {ma} clear of the guard band")

    def matrix(self, *params):
        a, L, nids = self.args(*params), self.ctx.L, C.c_longlong(-1)
        n = self.ctx._chk(L.l3d_affinity_matrix(*a, None, None, None, C.c_longlong(0), None, C.c_longlong(0), C.byref(nids)), "l3d_affinity_matrix")
        ei, ej, ew, l2g = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.float32), np.zeros(nids.value, np.int64)
        if n:
            assert L.l3d_affinity_matrix(*a, _p(ei), _p(ej), _p(ew), C.c_longlong(n), _p(l2g), C.c_longlong(len(l2g)), C.byref(nids)) == n
        return ei, ej, ew, l2g

    def edges(self, *params):
        a, L = self.args(*params), self.ctx.L
        n = self.ctx._chk(L.l3d_affinity_edges(*a, None, None, None, C.c_longlong(0)), "l3d_affinity_edges")
        gi, gj, w = np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros(n, np.float32)
        if n:
            assert L.l3d_affinity_edges(*a, _p(gi), _p(gj), _p(w), C.c_longlong(n)) == n
        return gi, gj, w

    def close(self):
        self.ctx.close()


def rel_gap(w32, w64):
    return float(np.max(np.abs(np.asarray(w32, np.float64) - w64) / w64, initial=0.0))


def check_matrix(run, r, got):
    """l3d_affinity_matrix's result `got` against the model's r: indices identical, weights within RTOL"""
    ei, ej, ew, l2g = got
    assert r.band == 0                                    # no similarity close enough to the threshold to flip in float32
    assert l2g.tolist() == [run.g(s) for s in r.l2g]
    assert np.array_equal(ei, r.ei) and np.array_equal(ej, r.ej)
    gap = rel_gap(ew, r.ew)
    assert gap <= RTOL
    WORST["gap"] = max(WORST["gap"], gap)
    WORST["chain"] = max(WORST["chain"], r.chain)


def check_edges(run, r, got, matrix_w):
    """l3d_affinity_edges' list against the model's candidates; the matrix's weights are those of the accepted candidates, bit for bit"""
    gi, gj, w = got
    assert gi.tolist() == [run.g(a) for a, _, _ in r.cand] and gj.tolist() == [run.g(b) for _, b, _ in r.cand]
    assert rel_gap(w, np.array([x[2] for x in r.cand])) <= RTOL
    assert np.array_equal(util.bits(w[r.acc]), util.bits(matrix_w[0::2]))


# ------------------------------------------------------------------------------------------------------------ fixtures
_runs = {}


def scene_run(name, perc=0.1):
    key = (name, perc)
    if key not in _runs:
        _runs[key] = Run(am.scene(name), perc=perc)
    return _runs[key]


@pytest.fixture(scope="module", autouse=True)
def _close_runs():
    yield
    for r in _runs.values():
        r.close()
    _runs.clear()


@functools.lru_cache(maxsize=None)
def exported(name, perc, collin):
    run = scene_run(name, perc)
    run.links(collin)
    return run.problem()


PROBLEMS = [(n, 0.1) for n in am.SCENES] + [("thirds", 0.3)]


# ------------------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("collin", COLLIN)
@pytest.mark.parametrize("name,perc", PROBLEMS)
def test_matrix_and_candidates_follow_model(name, perc, collin):
    run = scene_run(name, perc)
    pr = exported(name, perc, collin)
    run.links(collin)
    for params in PARAMS:
        params, r = run.settle(pr, *params)
        got = run.matrix(*params)
        check_matrix(run, r, got)
        check_edges(run, r, run.edges(*params), got[2])


def test_problems_reach_the_paths():
    """what the device problems reach, by the model on their exports (tests/test_affinity_model_cpu.py explains the paths none can)"""
    hits, chain = {p: 0 for p in am.PATHS}, 0
    for name, perc in PROBLEMS:
        for collin in COLLIN:
            pr = exported(name, perc, collin)
            for params in (DEFAULT, (200.0, 0.0, 0.5)):
                r = scene_run(name, perc).model(pr, *params)
                hits = {p: hits[p] + r.hits[p] for p in am.PATHS}
                chain = max(chain, r.chain)
    for p in am.PATHS:
        assert (hits[p] > 0) == (p not in ("direct_by_slink", "tlink_by_slink", "slink_by_direct", "slink_by_tlink")), p
    assert chain >= 4


def test_ref_cpu_append_order():
    """match_pairs_f64: the kept lists are in the reference's append order, not sorted by target"""
    run = Run(am.scene("overlap"), f64=True)
    try:
        run.links(5.0)
        pr = run.problem()
        assert any(lst != sorted(lst) for lst in pr.kept.values())
        for params in (DEFAULT, (20.0, 0.5, 0.2)):
            params, r = run.settle(pr, *params)
            got = run.matrix(*params)
            check_matrix(run, r, got)
            check_edges(run, r, run.edges(*params), got[2])
    finally:
        run.close()


def test_shuffled_view_order():
    """emission follows camID order, not the order of the l3d_set_views array"""
    sc = am.scene("thirds")
    run = Run(sc, order=np.random.default_rng(5).permutation(sc.num_views))
    try:
        assert not np.array_equal(run.order, np.sort(run.order))
        for collin in (-1.0, 5.0):
            run.links(collin)
            pr = run.problem()
            params, r = run.settle(pr, *DEFAULT)
            got = run.matrix(*params)
            check_matrix(run, r, got)
            check_edges(run, r, run.edges(*params), got[2])
    finally:
        run.close()


def test_degenerate_views():
    """a view with no segments, one with a single segment, views without estimates; then min_affinity above every similarity"""
    sc = am.scene("whole_broken")
    sc.segs[3] = np.zeros((0, 4), np.float32)
    sc.segs[6] = sc.segs[6][:1].copy()
    run = Run(sc)
    try:
        run.links(5.0)
        pr = run.problem()
        assert len(set(pr.views) - set(pr.est_cam.tolist())) >= 2          # views 3 and 6 (at least) have no estimates
        for params in (DEFAULT, (20.0, 0.0, 0.2)):
            params, r = run.settle(pr, *params)
            got = run.matrix(*params)
            check_matrix(run, r, got)
            check_edges(run, r, run.edges(*params), got[2])
        # nothing passes: similarities are at most 1
        L, nids = run.ctx.L, C.c_longlong(-1)
        a = run.args(200.0, 1.0, 1.0)
        assert L.l3d_affinity_edges(*a, None, None, None, C.c_longlong(0)) == 0
        assert L.l3d_affinity_matrix(*a, None, None, None, C.c_longlong(0), None, C.c_longlong(0), C.byref(nids)) == 0 and nids.value == 0
        buf_i, buf_j, buf_w = np.zeros(4, np.int32), np.zeros(4, np.int32), np.zeros(4, np.float32)
        assert L.l3d_rdd_affinity(run.ctx.h, 10, _p(buf_i), _p(buf_j), _p(buf_w), C.c_longlong(4)) == 0
    finally:
        run.close()


def test_links_on_with_empty_lists_is_links_off():
    run = Run(synth.make_scene(8, 300, 31, "ring2"))
    try:
        run.links(-1.0)
        off_m, off_e = run.matrix(*DEFAULT), run.edges(*DEFAULT)
        run.links(1e-4)
        assert run.ctx.L.l3d_collinear_total(run.ctx.h) == 0
        on_m, on_e = run.matrix(*DEFAULT), run.edges(*DEFAULT)
        assert len(off_m[0]) > 1000
        for a, b in zip(off_m + off_e, on_m + on_e):
            assert a.dtype == b.dtype and a.tobytes() == b.tobytes()
    finally:
        run.close()


def test_large_problem():
    """60 views x 1500 segments with links at 5 px: more than 1e5 candidates, long runs of one pair in the sort"""
    sc = am.pieces_scene(60, 1500, 96, "ring10", [am.HALVES, None, am.THIRDS, [(0.0, 1.0)]], 5, 4)
    run = Run(sc)
    try:
        run.links(5.0)
        pr = run.problem()
        params = DEFAULT
        # about 1e6 similarities: every window of 2e-5 around min_affinity holds some, so the decisions on those come from the
        # device's candidate list (a passing similarity is a candidate whenever its parent passes); the bookkeeping is the model's
        gi, gj, _ = run.edges(*params)
        seg = {run.g((int(c), s)): (int(c), s) for c in pr.views for s in range(run.nseg[run.pos[int(c)]])}
        listed = {(seg[a], seg[b]) for a, b in zip(gi.tolist(), gj.tolist())}
        near = am.restate(pr, *run.model_args(*params)).near
        r = am.restate(pr, *run.model_args(*params), decided={q: q in listed for q in near})
        print(f"\nlarge problem: {len(r.cand)} candidates, {len(r.ei) // 2} edges, chain {r.chain}, {len(near)} similarities in the guard band")
        assert len(r.cand) > 100000
        got = run.matrix(*params)
        check_matrix(run, r, got)
        check_edges(run, r, run.edges(*params), got[2])
    finally:
        run.close()


def test_cache_and_invalidation():
    run = Run(am.scene("overlap"))
    try:
        run.links(5.0)
        pr = run.problem()
        p1, r1 = run.settle(pr, *DEFAULT)
        p2, r2 = run.settle(pr, 20.0, 0.5, 0.2)
        first = run.matrix(*p1)
        check_matrix(run, r1, first)
        same = lambda got: all(a.tobytes() == b.tobytes() for a, b in zip(got, first))
        # candidates under other parameters leave the cached matrix alone
        gi, gj, w = run.edges(*p2)
        assert gi.tolist() == [run.g(a) for a, _, _ in r2.cand]
        assert same(run.matrix(*p1))
        # another matrix, then the first again: recomputed, the same
        check_matrix(run, r2, run.matrix(*p2))
        assert same(run.matrix(*p1))
        # new median depths with the same parameters: the model's new result, not the cached one
        md = run.md.copy()
        run.md = (md * np.float32(1.5)).astype(np.float32)
        run.ctx.update_view_params(run.descs(run.md))
        pr_md = run.problem()
        r_md = run.model(pr_md, *p1)
        got = run.matrix(*p1)
        check_matrix(run, r_md, got)
        assert not same(got)
        run.md = md
        run.ctx.update_view_params(run.descs(run.md))
        # links off and on again under the same parameters
        run.links(-1.0)
        check_matrix(run, run.model(run.problem(), *p1), run.matrix(*p1))
        run.links(5.0)
        assert same(run.matrix(*p1))
    finally:
        run.close()


def test_min_affinity_domain():
    """a negative or NaN min_affinity is rejected by both calls, and the rejected call leaves no affinity matrix behind"""
    run = Run(synth.make_scene(6, 200, 11, "ring2", collinear=True))
    try:
        L, h, nids = run.ctx.L, run.ctx.h, C.c_longlong(-1)
        buf_i, buf_j, buf_w = np.zeros(1 << 16, np.int32), np.zeros(1 << 16, np.int32), np.zeros(1 << 16, np.float32)
        rdd = lambda: L.l3d_rdd_affinity(h, 10, _p(buf_i), _p(buf_j), _p(buf_w), C.c_longlong(len(buf_i)))
        for bad in (-0.1, float("nan"), -0.0 - 1e-30):
            assert len(run.matrix(*DEFAULT)[0]) > 0 and rdd() > 0
            a = (h, C.c_float(200.0), C.c_float(run.median()), C.c_float(bad))
            assert L.l3d_affinity_matrix(*a, None, None, None, C.c_longlong(0), None, C.c_longlong(0), C.byref(nids)) == -1    # L3D_ERR_INVALID
            assert rdd() == -3                                                                                              # L3D_ERR_STATE
            assert len(run.matrix(*DEFAULT)[0]) > 0 and rdd() > 0
            assert L.l3d_affinity_edges(*a, None, None, None, C.c_longlong(0)) == -1
            assert rdd() == -3
        # zero is in the domain
        assert L.l3d_affinity_edges(h, C.c_float(200.0), C.c_float(run.median()), C.c_float(0.0), None, None, None, C.c_longlong(0)) > 0
    finally:
        run.close()


def test_report():
    """the worst weight gap against the model and the longest dependency chain of the problems above (pytest -s shows them)"""
    print(f"\naffinity vs float64 model: worst relative weight gap {WORST['gap']:.3g}, longest dependency chain {WORST['chain']}")
    assert WORST["gap"] <= RTOL
