"""The matcher on rows of thousands of matches (tests/crowded_rows.py): every kNN regime of the top-k key lists (kNN <= 16: top_rank,
17..31: rank_in_row, 32: the list never shrinks, > 32: keep-all then k_sort_rows' cut), keep-all at kNN 0 and -1, and k_sort_rows at
4, 2 and 1 warps per block with its grid-stride loop, under REF_GPU and REF_CPU semantics.  Every record is compared byte for byte, in
order, with rows derived in numpy from the oracle's keep-all rows: best first with the smaller tgt_seg first on a tie (kNN > 0),
ascending tgt_seg (kNN <= 0); REF_GPU depths are those l3d_match_dense computes for the same cells.  Also: the 8533-match row limit, candidate lists of every target, repeat calls and a gathered two-context job."""
import numpy as np
import pytest

from line3dpp_b200 import capi
from tests import crowded_rows as cr

pytestmark = pytest.mark.gpu

FIELDS = ("tgt_seg", "overlap", "d_p1", "d_p2", "d_q1", "d_q2")
L3D_ERR_UNSUPPORTED, L3D_ERR_STATE = -4, -3
LIMIT_MSG = "a row with more than 8533 matches (kNN <= 0 or kNN > 32)"


@pytest.fixture(scope="module")
def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def knn_job():
    return cr.knn_job()


@pytest.fixture(scope="module")
def band_jobs(num_sms):
    """one job per k_sort_rows band: its padding rows alone exceed what one sweep of the grid covers (num_sms * 16 blocks of
    `warps` rows), so the crowded rows after them are sorted by a later iteration of the grid-stride loop"""
    return {n: cr.band_job(n, pad_rows=num_sms * cr.GRID_BLOCKS_PER_SM * w + 1) for n, w in cr.SORT_BANDS.items()}


def _match(ctx, job, sem, knn, pairs=None):
    pairs = job.pairs if pairs is None else pairs
    from tests import util
    ctx.set_views(util.scene_descs(job.scene), job.scene.segs)
    if sem == "gpu":
        ctx.match_pairs(pairs, util.pair_F(job.scene, pairs), cr.EPI, knn)
    else:
        ctx.match_pairs_f64(pairs, _F64(job.scene, pairs), cr.EPI, knn)


def _F64(scene, pairs):
    return np.stack([cr.synth.fundamental(scene.K[s], scene.R[s], scene.t[s], scene.K[t], scene.R[t], scene.t[t]).reshape(9) for s, t in pairs])


def _rows(ctx, job, pairs=None):
    """(counts, records up to each row's count, concatenated) of every pair"""
    pairs = job.pairs if pairs is None else pairs
    out = []
    for p, (s, _t) in enumerate(pairs):
        counts, recs = ctx.pair_matches(p, len(job.scene.segs[s]))
        keep = np.arange(recs.shape[1])[None, :] < counts[:, None]
        out.append((counts.copy(), recs[keep].copy()))
    return out


def _same_rows(a, b):
    assert len(a) == len(b)
    for p, ((ca, ra), (cb, rb)) in enumerate(zip(a, b)):
        assert ca.tobytes() == cb.tobytes(), p
        for f in FIELDS:
            assert np.ascontiguousarray(ra[f]).tobytes() == np.ascontiguousarray(rb[f]).tobytes(), (p, f)


def _dense_depths(ctx, job, p, counts, recs):
    """REF_GPU: the oracle's keep-all records with the depths l3d_match_dense computes for the same cells.  The oracle's float
    restatement normalises with 1 / sqrtf where the device uses rsqrtf, so its depths differ in the last bits (tests/test_match_gpu.py
    pins it to 1e-5 relative); l3d_match_dense is pinned bit for bit to the reference's kernel, and k_match_topk / k_match_cand form
    their depths with the same exact_depths on the same cached rays."""
    from tests import util
    s, t = job.pairs[p]
    dep, ov = ctx.match_dense(s, t, util.pair_F(job.scene, job.pairs[p:p + 1])[0], cr.EPI, len(job.scene.segs[s]), len(job.scene.segs[t]))
    recs = recs.copy()
    for r in np.flatnonzero(counts):
        e = recs[r, :counts[r]]
        j = e["tgt_seg"].astype(np.int64)
        assert ov[r, j].tobytes() == e["overlap"].tobytes()
        d = dep[r, j]
        for i, f in enumerate(("d_p1", "d_p2", "d_q1", "d_q2")):
            assert np.all(np.abs(d[:, i] - e[f]) <= 1e-5 * np.abs(d[:, i]))
            e[f] = d[:, i]
        recs[r, :counts[r]] = e
    return recs


def _check(ctx, job, sem, knn):
    """counts and records of every row as expected_rows derives them from the oracle's keep-all rows (REF_GPU: with the depths of
    l3d_match_dense), in order, byte for byte"""
    got = _rows(ctx, job)
    matches = 0
    for p, (counts, recs) in enumerate(job.keep_all[sem]):
        if sem == "gpu":
            recs = _dense_depths(ctx, job, p, counts, recs)
        ec, er = cr.expected_rows(counts, recs, knn)
        gc, gr = got[p]
        assert np.array_equal(gc, ec), (sem, knn, p, np.flatnonzero(gc != ec)[:5])
        off = np.concatenate([[0], np.cumsum(gc)])
        for r in np.flatnonzero(ec):
            g = gr[off[r]:off[r + 1]]
            for f in FIELDS:
                assert np.ascontiguousarray(g[f]).tobytes() == np.ascontiguousarray(er[r][f]).tobytes(), (sem, knn, p, r, f)
        matches += int(ec.sum())
    return got, matches


@pytest.mark.parametrize("sem", ["gpu", "cpu"])
@pytest.mark.parametrize("knn", cr.KNNS)
def test_crowded_rows_every_knn(gpu_ctx, knn_job, sem, knn):
    _match(gpu_ctx, knn_job, sem, knn)
    assert gpu_ctx.L.l3d_match_stride(gpu_ctx.h) == (knn if 0 < knn <= 32 else knn_job.longest)
    _, matches = _check(gpu_ctx, knn_job, sem, knn)
    assert matches > (10000 if knn <= 0 else min(knn, 60) * 30)


@pytest.mark.parametrize("sem", ["gpu", "cpu"])
@pytest.mark.parametrize("knn", [0, 100])
@pytest.mark.parametrize("longest", list(cr.SORT_BANDS))
def test_sort_shapes(gpu_ctx, band_jobs, num_sms, sem, knn, longest):
    """k_sort_rows at the edges of its 4-, 2- and 1-warp shapes, with more rows than one sweep of its grid"""
    job = band_jobs[longest]
    warps = cr.SORT_BANDS[longest]
    assert cr.sort_warps(longest) == warps
    _match(gpu_ctx, job, sem, knn)
    assert gpu_ctx.L.l3d_match_stride(gpu_ctx.h) == longest
    sweep = num_sms * cr.GRID_BLOCKS_PER_SM * warps            # rows one sweep of the grid sorts
    assert gpu_ctx.match_total_rows() > sweep and len(job.scene.segs[0]) >= sweep   # the crowded rows come after the padding rows
    _check(gpu_ctx, job, sem, knn)


@pytest.mark.parametrize("sem", ["gpu", "cpu"])
def test_row_limit(gpu_ctx, knn_job, sem):
    """a row of 8534 matches fails keep-all and kNN > 32 with the limit in the message, leaves no result, and the next call works"""
    job = cr.band_job(cr.ROW_LIMIT + 1, pad_rows=8)
    assert job.longest == 8534
    for knn in (0, 40):
        with pytest.raises(capi.L3DError, match=rf"failed \({L3D_ERR_UNSUPPORTED}\)") as e:
            _match(gpu_ctx, job, sem, knn)
        assert LIMIT_MSG in str(e.value) and LIMIT_MSG in gpu_ctx.L.l3d_last_error(gpu_ctx.h).decode()
        assert gpu_ctx.match_total_rows() == -1
        assert gpu_ctx.L.l3d_match_stride(gpu_ctx.h) == L3D_ERR_STATE
        _match(gpu_ctx, knn_job, sem, knn)
        _check(gpu_ctx, knn_job, sem, knn)


@pytest.mark.parametrize("sem", ["gpu", "cpu"])
def test_candidates_equal_the_scan(gpu_ctx, knn_job, sem):
    """every target of every crowded pair, in both camera orders, as candidates: shuffled and duplicated, the rows are the scan's"""
    pairs = np.concatenate([knn_job.pairs, knn_job.pairs[:, ::-1]]).astype(np.int32)
    rng = np.random.default_rng(5)
    trip = []
    for p, (s, t) in enumerate(pairs):
        a, b = np.meshgrid(np.arange(len(knn_job.scene.segs[s])), np.arange(len(knn_job.scene.segs[t])), indexing="ij")
        trip.append(np.stack([np.full(a.size, p), a.ravel(), b.ravel()], 1))
    trip = np.concatenate(trip + [trip[0][::3], trip[-1][::7]])
    trip = np.ascontiguousarray(trip[rng.permutation(len(trip))], np.int32)
    from tests import util
    for knn in cr.KNNS:
        _match(gpu_ctx, knn_job, sem, knn, pairs)
        want = _rows(gpu_ctx, knn_job, pairs)
        stride = gpu_ctx.L.l3d_match_stride(gpu_ctx.h)
        F = util.pair_F(knn_job.scene, pairs) if sem == "gpu" else _F64(knn_job.scene, pairs)
        gpu_ctx.match_pairs_cand(pairs, F, np.ones(len(pairs), np.int32), trip, cr.EPI, knn, f64=sem == "cpu")
        assert gpu_ctx.L.l3d_match_stride(gpu_ctx.h) == stride
        _same_rows(_rows(gpu_ctx, knn_job, pairs), want)


@pytest.mark.parametrize("knn", [-1, 100])
def test_repeat_is_byte_identical(gpu_ctx, knn_job, knn):
    """Store writes rows in arrival order; after the sort two identical calls agree byte for byte"""
    runs = []
    for _ in range(2):
        _match(gpu_ctx, knn_job, "gpu", knn)
        runs.append(_rows(gpu_ctx, knn_job))
    _same_rows(runs[0], runs[1])


@pytest.mark.parametrize("knn", [0, 100])
def test_gathered_shards_equal_one_context(knn_job, knn):
    """two contexts on one device match disjoint pair ranges whose own strides fall in different k_sort_rows bands (4 and 1 warps);
    gathered, they give the single context's rows, stride included"""
    from tests import util
    job = cr.build(cr.knn_rows()[:2] + [[cr.Row("distinct", 4267), cr.Row("tie", 300)]], seed=303)
    F = util.pair_F(job.scene, job.pairs)
    P = len(job.pairs)
    ctxs = [capi.Context(0) for _ in range(3)]
    try:
        for c in ctxs:
            c.set_views(util.scene_descs(job.scene), job.scene.segs)
        ctxs[0].match_pairs(job.pairs, F, cr.EPI, knn)
        want = _rows(ctxs[0], job)
        want_stride = ctxs[0].L.l3d_match_stride(ctxs[0].h)
        ctxs[1].match_pairs_range(job.pairs, F, 0, P - 1, cr.EPI, knn)
        ctxs[2].match_pairs_range(job.pairs, F, P - 1, P, cr.EPI, knn)
        own = [c.L.l3d_match_stride(c.h) for c in ctxs[1:]]
        assert [cr.sort_warps(s) for s in own] == [4, 1], own
        ctxs[1].match_gather(ctxs[1:], [0, P - 1, P])
        ctxs[1].sync()
        assert ctxs[1].L.l3d_match_stride(ctxs[1].h) == want_stride == 4267
        _same_rows(_rows(ctxs[1], job), want)
        _check(ctxs[1], job, "gpu", knn)
    finally:
        for c in ctxs:
            c.close()
