"""The scoring sweep (l3d_score_sweep, csrc/l3d_pipeline.cu) on scenes wide enough that its tables outgrow shared memory and are
read from global memory instead: views with more than 64 neighbour chunks, more than 512 chunk boundaries per CTA, segments with
more than 192 entries, lists longer than the shared-memory staging capacity; and segments matched into more than 48 target
cameras.  The other suites never cross these thresholds (at most 25 chunks per view).

  W1  70 views, dense neighbours (np = 69), REF_GPU: chunk descriptors and chunk-sort keys read from global memory
  W2  64 views, ring +-30 (np = 60), REF_GPU: chunk boundaries in shared memory up to 8 segments per CTA, in global memory from 9 on
  W3  W2 with a heavy tail (one segment matched by 120 pieces of its line in each of 41 views): the automatic geometry
      overflows the staging capacity and scores that CTA out of the global scratch
  W4  52 views, dense (np = 51), REF_CPU: segments with more than 48 target cameras (the per-camera maximum beyond the 48-slot map)

Every test first asserts, from what the product exports, that the threshold it is about is crossed (np from the pair list; the
active entries of a segment are a lower bound of its list length), so none of them can pass without crossing it.
The verbatim reference's results are stored in tests/golden/ref_gpu_wide_v1.npz (REF_GPU, W1-W3) and
tests/golden/ref_full_wide_cpu_v1.npz (REF_CPU, W4), made by tests/golden/make_ref_wide_golden.py."""
import ctypes as C
import os

import numpy as np
import pytest

from line3dpp_b200 import capi, line3d, synth
from tests import util

pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GPU_GOLDEN = os.path.join(G, "ref_gpu_wide_v1.npz")
CPU_GOLDEN = os.path.join(G, "ref_full_wide_cpu_v1.npz")

# the sweep's capacity thresholds (csrc/l3d_pipeline.cu): beyond them a table is read from global instead of shared memory
SW_MAXCH = 512            # chunk boundaries per CTA held in shared memory
SW_MAXNP = 64             # chunk descriptors held in shared memory
CS_MAXN = 192             # entries of one segment the chunk sort handles in shared memory
SC_MAP = 48               # target cameras of the REF_CPU per-camera maximum map
CAP_MAX = {False: 4096, True: 2048}       # entries staged in shared memory per CTA at most (REF_GPU, REF_CPU)
FORCED_SEGS = (1, 2, 7, 8, 9, 16)         # L3D_SW_SEGS settings of the geometry-invariance test

# name: (views, segments per view, neighbours, kNN, diffusion); the scene itself is wide_scene(name)
WIDE = {"w1": (70, 150, "dense", 10, False), "w2": (64, 150, "ring30", 10, True), "w3": (64, 150, "ring30", 10, False),
        "w4": (52, 90, "dense", 4, False)}
SEED = 5
W3_PIECES = 120
NSAMPLE = 4000            # affinity weights stored per scene


def _observers(sc, line, tgt):
    return [v for v in range(sc.num_views) if v != tgt and line in set(sc.line_ids[v].tolist()) and tgt in set(sc.neighbors[v].tolist())]


def _heavy_tail(sc, pieces):
    """the last view's segment whose 3D line the most neighbours observe is matched by `pieces` pieces of their segment of that
    line in each of them: its list is far longer than its view's mean.  Returns its index.
    The pieces are random sub-intervals (start in the first quarter, end in the last), not copies: identical or merely shifted
    copies tie in the kNN lists of the rows that match into them (equal overlaps, e.g. all pieces inside the epipolar band of a
    longer row), and the reference's order among equal overlaps is unspecified.  Pieces of different lengths never tie."""
    tgt = sc.num_views - 1
    seg = max(range(len(sc.segs[tgt])), key=lambda i: (len(_observers(sc, sc.line_ids[tgt][i], tgt)), -i))
    line = sc.line_ids[tgt][seg]
    for v in _observers(sc, line, tgt):
        j = int(np.flatnonzero(sc.line_ids[v] == line)[0])
        s = sc.segs[v][j].astype(np.float64)
        rng = np.random.default_rng([SEED, v])
        u, w = rng.uniform(0.0, 0.25, (pieces, 1)), rng.uniform(0.75, 1.0, (pieces, 1))
        sub = np.concatenate([s[:2] + u * (s[2:] - s[:2]), s[:2] + w * (s[2:] - s[:2])], axis=1).astype(np.float32)
        sc.segs[v] = np.insert(sc.segs[v], j, sub.reshape(-1, 4), axis=0)
        sc.line_ids[v] = np.insert(sc.line_ids[v], j, np.full(pieces, line))
    return seg


def _shifted(s, px):
    """segment s moved by px pixels along its normal"""
    d = np.array([s[2] - s[0], s[3] - s[1]], np.float64)
    n = np.array([-d[1], d[0]]) / np.linalg.norm(d) * px
    return np.array([s[0] + n[0], s[1] + n[1], s[2] + n[0], s[3] + n[1]], np.float32)


def _near_triples(sc, views):
    """in `views`, every segment of a 3D line view 0 also observes becomes three parallel segments, 1.5 px off, exact, 0.7 px
    off: three positive similarities per target camera in the order low, high, middle.  View 0's lists reach these cameras after
    48 others, so the REF_CPU per-camera maximum of these cameras is the one recovered outside the 48-slot map."""
    seen0 = set(sc.line_ids[0].tolist())
    for v in views:
        segs, ids = [], []
        for s, ln in zip(sc.segs[v], sc.line_ids[v]):
            trip = [_shifted(s, 1.5), s, _shifted(s, 0.7)] if int(ln) in seen0 else [s]
            segs += trip
            ids += [ln] * len(trip)
        sc.segs[v], sc.line_ids[v] = np.ascontiguousarray(segs, np.float32), np.array(ids)


def wide_scene(name):
    V, N, nb, _, _ = WIDE[name]
    sc = synth.make_scene(V, N, SEED, nb)
    if name == "w3":
        _heavy_tail(sc, W3_PIECES)
    if name == "w4":
        _near_triples(sc, (V - 3, V - 2, V - 1))
    return sc


def heavy_segment(sc):
    """W3: the segment of the last view made heavy by _heavy_tail (recomputed on the unmodified scene)"""
    V, N, nb, _, _ = WIDE["w3"]
    return _heavy_tail(synth.make_scene(V, N, SEED, nb), 0)


# ---------------------------------------------------------------------------------------------------------- preconditions
def chunks_per_view(L, V):
    """np: the number of view pairs that involve each view"""
    return np.bincount(L.pairs().reshape(-1), minlength=V)


def active_per_segment(L, sc, cam):
    return np.bincount(L.view_matches(cam, False)["src_seg"].astype(np.int64), minlength=len(sc.segs[cam]))


def max_cta_entries(counts, segs):
    """the most active entries a CTA of `segs` consecutive segments holds (a lower bound of what it stages)"""
    return max(int(counts[s:s + segs].sum()) for s in range(0, len(counts), segs))


def max_target_cameras(L, cam):
    m = L.view_matches(cam, False)
    best = 0
    for s in np.unique(m["src_seg"]):
        best = max(best, len(np.unique(m["tgt_cam"][m["src_seg"] == s])))
    return best


# ---------------------------------------------------------------------------------------------------------- runs
def run(monkeypatch, sc, name, segs=None, cpu_sem=False, reconstruct=False):
    """the product's pipeline on scene `sc`; segs: L3D_SW_SEGS (segments per CTA of the sweep), None: the automatic choice"""
    if segs is None:
        monkeypatch.delenv("L3D_SW_SEGS", raising=False)
    else:
        monkeypatch.setenv("L3D_SW_SEGS", str(segs))
    _, _, _, knn, diffusion = WIDE[name]
    L = line3d.Line3D(neighbors_by_worldpoints=False, use_gpu=not cpu_sem)
    L.add_scene(sc)
    L.match_images(knn=knn)
    if reconstruct:
        L.reconstruct_3d_lines(3, diffusion)
    return L


def sweep_record(L, sc):
    """every view's scored and kept list (all fields, score3D bits included) and the estimates, as digests"""
    out = [(util.match_sha(L.view_matches(cam, False)), util.match_sha(L.view_matches(cam, True))) for cam in sc.cam_ids]
    best, p = L.estimates()
    return out, util.match_sha(best), util.sha(np.ascontiguousarray(p))


@pytest.fixture(scope="module")
def scenes():
    return {name: wide_scene(name) for name in WIDE}


@pytest.fixture(scope="module")
def gpu_golden():
    return np.load(GPU_GOLDEN)


def check_ref_gpu_preconditions(name, L, sc):
    npv = chunks_per_view(L, sc.num_views)
    counts = [active_per_segment(L, sc, cam) for cam in sc.cam_ids]
    longest = max(int(c.max()) for c in counts)
    if name == "w1":
        assert (npv > SW_MAXNP).all(), npv            # chunk descriptors and chunk-sort keys read from global memory
    else:
        assert (npv <= SW_MAXNP).all() and (8 * npv <= SW_MAXCH).all() and (9 * npv > SW_MAXCH).all(), npv
    assert longest > CS_MAXN, longest                 # chunk-sort keys read from global memory
    if name == "w3":
        # the heavy segment alone holds more than any CTA can stage, whatever geometry the sweep picks: global scratch
        n = int(counts[-1][heavy_segment(sc)])
        assert n > CAP_MAX[False], n


@pytest.mark.parametrize("name", ["w1", "w2", "w3"])
def test_ref_gpu_wide_vs_verbatim_reference(monkeypatch, scenes, gpu_golden, name):
    """W1-W3 with the automatic geometry against the verbatim reference pipeline on the GPU, every stage
    (tests/test_ref_full_gpu.py:compare_all_stages: lists and score3D bit for bit, estimates to 1e-12, local ids, affinity
    edges, clusters, 3D end points to 1e-6)"""
    from tests.test_ref_full_gpu import compare_all_stages
    sc = scenes[name]
    L = run(monkeypatch, sc, name, reconstruct=True)
    check_ref_gpu_preconditions(name, L, sc)
    total, nedges, nlines = compare_all_stages(L, gpu_golden, name + "_", sc.cam_ids, [len(s) for s in sc.segs], -1.0)
    assert total > 100000 and nedges > 1000 and nlines > 100, (total, nedges, nlines)
    L.close()


@pytest.mark.parametrize("name", ["w1", "w2", "w3", "w4"])
def test_sweep_geometry_invariance(monkeypatch, scenes, name):
    """the segments per CTA (L3D_SW_SEGS) move every view across the shared / global boundaries of the chunk tables and of the
    staged entries; none of that may change a bit of the scored and kept lists, score3D or the estimates"""
    sc = scenes[name]
    cpu_sem = name == "w4"
    L = run(monkeypatch, sc, name, cpu_sem=cpu_sem)
    auto = sweep_record(L, sc)
    npv = chunks_per_view(L, sc.num_views)
    counts = [active_per_segment(L, sc, cam) for cam in sc.cam_ids]
    L.close()
    # the settings cover both sides of every boundary
    assert any((s * npv <= SW_MAXCH).all() for s in FORCED_SEGS) and any((s * npv > SW_MAXCH).all() for s in FORCED_SEGS), npv
    # global scratch in two consecutive views (the sweep runs them in ascending camID, two kernels may be in flight and share
    # the double-buffered scratch): a CTA of each holds more entries than any CTA stages in shared memory
    over = [max_cta_entries(c, max(FORCED_SEGS)) > CAP_MAX[cpu_sem] for c in counts]
    assert any(a and b for a, b in zip(over, over[1:])), over
    for segs in FORCED_SEGS:
        L = run(monkeypatch, sc, name, segs=segs, cpu_sem=cpu_sem)
        rec = sweep_record(L, sc)
        L.close()
        for cam in sc.cam_ids:
            assert rec[0][cam][0].tobytes() == auto[0][cam][0].tobytes(), f"L3D_SW_SEGS={segs}: scored list of view {cam}"
            assert rec[0][cam][1].tobytes() == auto[0][cam][1].tobytes(), f"L3D_SW_SEGS={segs}: kept list of view {cam}"
        assert rec[1].tobytes() == auto[1].tobytes() and rec[2].tobytes() == auto[2].tobytes(), f"L3D_SW_SEGS={segs}: estimates"


# ---------------------------------------------------------------------------------------------------------- REF_CPU, W4
def check_w4_preconditions(L, sc):
    npv = chunks_per_view(L, sc.num_views)
    assert (npv == sc.num_views - 1).all(), npv
    ncam = max(max_target_cameras(L, cam) for cam in sc.cam_ids[:4])
    assert ncam >= SC_MAP + 2, ncam                   # the per-camera maximum beyond the 48-slot map


W4_U_MAX = 8               # |U| of W4: 4 segments whose two best kept scores lie within their bound E of each other (measured)


@pytest.fixture(scope="module")
def w4_model(scenes, oracle):
    """the oracle's REF_CPU run of W4 and the float64 model on it (tests/refcpu_model.py)"""
    from tests import refcpu_model as rm
    sc = scenes["w4"]
    P = oracle.OraclePipeline(False, False)
    P.add_scene(sc)
    oracle.set_threads(os.cpu_count() or 1)
    P.match_images(knn=WIDE["w4"][3])
    oracle.set_threads(1)
    cams = rm.Cameras.of_scene(sc, [P.view_info(c)[0] for c in sc.cam_ids])
    return (P,) + rm.run_model(cams, P, sc.cam_ids, 200.0)


def test_refcpu_wide_vs_oracle(monkeypatch, scenes, w4_model):
    """W4, REF_CPU semantics, against the oracle's restatement of matchingCPU + scoringCPU: every difference accounted for by the
    float64 model (tests/refcpu_model.py).  Outside U: lists, order and depths identical, score3D within the per-entry bound E,
    kept sets, best matches and estimates exact; so a wrong per-camera maximum on the segments that reach past 48 cameras
    changes a score by far more than E and fails."""
    from tests import refcpu_model as rm
    sc = scenes["w4"]
    L = run(monkeypatch, sc, "w4", cpu_sem=True)
    check_w4_preconditions(L, sc)
    _, res, scored, kept, est = w4_model
    print("W4 |U| =", res.size(), res.events())
    assert res.size() <= W4_U_MAX, res.events()
    st = rm.check_run(res, scored, kept, est, lambda c: L.view_matches(c, False), lambda c: L.view_matches(c, True), L.estimates())
    assert st["entries"] > 50000, st
    L.close()


def test_refcpu_wide_vs_verbatim_cpu_reference_golden(monkeypatch, scenes, w4_model):
    """W4, REF_CPU semantics, against the verbatim CPU reference (tests/golden/ref_full_wide_cpu_v1.npz).  U comes from the live
    oracle on the same inputs (the oracle restates the verbatim reference: tests/test_ref_full_cpu.py): a view's scored list may
    differ from the golden digest only where U holds an uncertain list entry, its kept count only where U reaches a kept
    decision, and the line count by at most one per segment whose kept set or estimate U reaches (such a segment joins or
    leaves one cluster)."""
    from tests import refcpu_model as rm
    from tests.test_ref_full_cpu import digest_matches
    z = np.load(CPU_GOLDEN)
    sc = scenes["w4"]
    L = run(monkeypatch, sc, "w4", cpu_sem=True)
    check_w4_preconditions(L, sc)
    assert np.array_equal(L.pairs(), z["pairs"])
    _, res, _, _, _ = w4_model
    assert res.size() <= W4_U_MAX, res.events()
    for cam in sc.cam_ids:
        m = L.view_matches(cam, kept_only=False)
        same = len(m) == int(z[f"scored_n_{cam}"][0]) and np.array_equal(digest_matches(m), z[f"scored_sha_{cam}"])
        assert same or res.gone.get(cam) or res.phantom.get(cam) or res.views[cam].ties, f"view {cam}: scored list differs and U holds none of it"
        nk = len(L.view_matches(cam, kept_only=True))
        assert nk == int(z[f"kept_n_{cam}"][0]) or res.views[cam].kept_u, f"view {cam}: kept count {nk} outside U"
    L.reconstruct_3d_lines(3, False)
    nl, nl_ref = L.stats()["lines3D"], int(z["num_lines"][0])
    assert nl_ref > 100 and abs(nl - nl_ref) <= rm.kept_decisions(res), (nl, nl_ref, rm.kept_decisions(res))
    L.close()


# ---------------------------------------------------------------------------------------------------------- l3d_argsort_f32
def argsort_f32(ctx, keys):
    keys = np.ascontiguousarray(keys, np.float32)
    perm = np.full(len(keys), 0xFFFFFFFF, np.uint32)
    rc = ctx.L.l3d_argsort_f32(ctx.h, C.c_longlong(len(keys)), capi._p(keys), capi._p(perm))
    return rc, perm


def tie_heavy_keys(n, seed):
    """the quantised weights of tests/golden/make_ref_cpu_golden.py:cluster_graphs: 23 values, many ties"""
    return np.random.default_rng(seed).choice(np.linspace(0.5, 1.0, 23), n).astype(np.float32)


def signed_zero_keys(n, seed):
    """+0.0 and -0.0 (equal under <: they keep their input order), denormals of both signs and a few ordinary values"""
    rng = np.random.default_rng(seed)
    tiny = np.float32(np.finfo(np.float32).smallest_subnormal)
    pool = np.array([0.0, -0.0, tiny, -tiny, 3 * tiny, np.float32(1e-39), np.float32(-1e-39), np.finfo(np.float32).tiny, 1.0, -1.0], np.float32)
    return pool[rng.integers(0, len(pool), n)]


@pytest.mark.parametrize("n", [0, 1, 2, 255, 256, 257, 4099, (1 << 20) + 3])
@pytest.mark.parametrize("kind", ["ties", "zeros_denormals", "uniform"])
def test_argsort_f32_vs_numpy_stable(gpu_ctx, n, kind):
    """performClustering's weight sort (std::list::sort with <: stable, ties in input order) against np.argsort(kind="stable")"""
    if kind == "ties":
        keys = tie_heavy_keys(n, n)
    elif kind == "zeros_denormals":
        keys = signed_zero_keys(n, n)
    else:
        keys = np.random.default_rng(n).normal(size=n).astype(np.float32)
    rc, perm = argsort_f32(gpu_ctx, keys)
    assert rc == 0, gpu_ctx.L.l3d_last_error(gpu_ctx.h)
    assert np.array_equal(perm, np.argsort(keys, kind="stable").astype(np.uint32))
    if kind == "zeros_denormals" and n > 2:
        z = perm[keys[perm] == 0]
        assert len(z) > 1 and (np.diff(z.astype(np.int64)) > 0).all()     # +0.0 / -0.0 in input order


L3D_ERR_INVALID = -1


def test_argsort_f32_argument_errors(gpu_ctx):
    """a negative count, a missing key or output array, or no context: L3D_ERR_INVALID, and nothing is written"""
    keys = np.ones(4, np.float32)
    perm = np.full(4, 7, np.uint32)
    L = gpu_ctx.L
    for args in ((gpu_ctx.h, C.c_longlong(-1), capi._p(keys), capi._p(perm)), (gpu_ctx.h, C.c_longlong(4), None, capi._p(perm)),
                 (gpu_ctx.h, C.c_longlong(4), capi._p(keys), None), (None, C.c_longlong(4), capi._p(keys), capi._p(perm))):
        assert L.l3d_argsort_f32(*args) == L3D_ERR_INVALID
        assert (perm == 7).all()
    assert b"l3d_argsort_f32" in L.l3d_last_error(gpu_ctx.h)
    assert L.l3d_argsort_f32(gpu_ctx.h, C.c_longlong(0), None, None) == 0       # nothing to sort
    rc, perm = argsort_f32(gpu_ctx, np.array([2.0, 1.0], np.float32))           # the context still works
    assert rc == 0 and list(perm) == [1, 0]
