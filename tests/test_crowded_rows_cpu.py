"""The crowded-row jobs of tests/crowded_rows.py reach what tests/test_match_crowded_gpu.py is named for, checked on the CPU oracle
alone: every row length in every kind under both semantics, the k_sort_rows band of every call's longest row, a tie across the k-th
place for every kNN, tie runs whose smallest index sits at an end of the run, and the derived top-k rows equal to the oracle's own
where no tie sits at the k-th place."""
import numpy as np
import pytest

from tests import crowded_rows as cr
from tests import util

SEMS = ("gpu", "cpu")


@pytest.fixture(scope="module")
def knn_job():
    return cr.knn_job()


@pytest.fixture(scope="module")
def band_jobs():
    return {n: cr.band_job(n, pad_rows=8) for n in (*cr.SORT_BANDS, cr.ROW_LIMIT + 1)}


def test_row_limit_is_the_sort_capacity():
    assert cr.ROW_LIMIT == 8533
    assert [cr.sort_warps(n) for n in (1, 2133, 2134, 4266, 4267, 8533, 8534)] == [4, 4, 2, 2, 1, 1, 0]


@pytest.mark.parametrize("sem", SEMS)
def test_every_length_in_every_kind(knn_job, sem):
    got = {}
    for p, rows in enumerate(knn_job.rows):
        counts = knn_job.keep_all[sem][p][0]
        for r, row in enumerate(rows):
            assert counts[r] == row.n
            got.setdefault(row.kind, set()).add(int(counts[r]))
    for kind in ("distinct", "tie", "tie_at_k"):
        assert set(cr.LENGTHS) <= got[kind], (kind, sorted(set(cr.LENGTHS) - got[kind]))
    assert {0, 1, 32, 33, 64, 200} <= set(cr.LENGTHS)
    assert all({k - 1, k, k + 1} <= set(cr.LENGTHS) for k in cr.TOPK)
    assert cr.sort_warps(knn_job.longest) == 4 and knn_job.longest > 2000


@pytest.mark.parametrize("sem", SEMS)
def test_overlaps_of_each_kind(knn_job, sem):
    """distinct rows: distinct overlaps; tie rows: one record repeated; every record in (epi, 1] with four positive depths"""
    for p, rows in enumerate(knn_job.rows):
        counts, recs = knn_job.keep_all[sem][p]
        for r, row in enumerate(rows):
            e = recs[r, :counts[r]]
            assert np.all(e["overlap"] > cr.EPI) and np.all(e["overlap"] <= 1.0)
            for f in ("d_p1", "d_p2", "d_q1", "d_q2"):
                assert np.all(e[f] > 0)
            if row.kind == "distinct":
                assert len(np.unique(e["overlap"])) == row.n
            elif row.kind == "tie" and row.n:
                assert len(np.unique(e["overlap"])) == 1 and len(np.unique(e["d_p1"])) == 1


@pytest.mark.parametrize("sem", SEMS)
def test_sort_bands_and_the_limit(band_jobs, sem):
    for n, job in band_jobs.items():
        longest = max(int(c.max(initial=0)) for c, _ in job.keep_all[sem])
        assert longest == n == job.longest
        assert cr.sort_warps(longest) == (cr.SORT_BANDS[n] if n in cr.SORT_BANDS else 0)
        assert job.rows[0][0].kind == "pad" and len(job.rows[0]) == 8         # the padding rows come first


@pytest.mark.parametrize("sem", SEMS)
def test_a_tie_straddles_every_k(knn_job, sem):
    for k in cr.TOPK:
        hits = 0
        for p, rows in enumerate(knn_job.rows):
            counts, recs = knn_job.keep_all[sem][p]
            _, er = cr.expected_rows(counts, recs, len(recs[0]))
            hits += sum(cr.tie_at(x, k) for x in er)
        assert hits > 0, k


def test_tie_runs_put_their_smallest_index_at_an_end(knn_job):
    """the run's targets in column order (the order of their arcs): its smallest index sits at one end, the next smallest at the other"""
    assert len(knn_job.runs) == sum(r.kind == "tie_at_k" and r.n > r.prefix for rows in knn_job.rows for r in rows)
    for run in knn_job.runs.values():
        s = sorted(run)
        assert run[-1] == s[0]
        if len(run) > 1:
            assert run[0] == s[1]


@pytest.mark.parametrize("sem", SEMS)
@pytest.mark.parametrize("knn", cr.TOPK)
def test_derived_top_k_is_the_oracles_where_no_tie_at_k(knn_job, oracle, sem, knn):
    fn = oracle.lib().orc_match_lines_f32 if sem == "gpu" else oracle.lib().orc_match_lines_f64
    F = knn_job.F32() if sem == "gpu" else knn_job.F64()
    RtKinv, C = cr.synth.camera_blocks(knn_job.scene)
    compared = 0
    for p, (s, t) in enumerate(knn_job.pairs):
        sc = knn_job.scene
        if sem == "gpu":
            pi = util.pair_inputs(sc, s, t)
            args = (pi["ls"], pi["lt"], pi["F"], pi["Rs"], pi["Rt"], pi["Cs"], pi["Ct"])
        else:
            args = (sc.segs[s], sc.segs[t], F[p], RtKinv[s].reshape(9), RtKinv[t].reshape(9), C[s], C[t])
        oc, oo, _, _ = oracle.match_lines(fn, *args, s, t, cr.EPI, knn, f64=sem == "cpu")
        counts, recs = knn_job.keep_all[sem][p]
        ec, er = cr.expected_rows(counts, recs, knn)
        _, full = cr.expected_rows(counts, recs, len(recs[0]))
        assert np.array_equal(oc, ec)
        for r in range(len(counts)):
            if cr.tie_at(full[r], knn):
                continue
            a = oo[r, :oc[r]]
            a = a[np.argsort(a["tgt_seg"])]
            b = er[r][np.argsort(er[r]["tgt_seg"])]
            for f in ("tgt_seg", "overlap", "d_p1", "d_p2", "d_q1", "d_q2"):
                assert a[f].tobytes() == b[f].tobytes(), (p, r, f)
            compared += oc[r] > 0
    assert compared > 40
