"""k_match_topk's work units: every instantiation (REF_GPU / REF_CPU semantics, top-k and keep-all) row by row against the CPU oracle
on pairs whose target view is exactly resident in the ring (3072 segments, one pass), holds one entry more (3073: the second pass
holds one entry) or takes three passes (6500).  Source views of 1, 191, 193 and 2500 rows give single, uneven and partial units on
both sides.  Rows reach the warps in an order that depends on timing, so two identical calls must also agree byte for byte."""
import numpy as np
import pytest

from line3dpp_b200 import synth
from tests import util

pytestmark = pytest.mark.gpu

NS = {0: 1, 1: 191, 2: 193, 3: 2500}
NT = {4: 3072, 5: 3073, 6: 6500}
PAIRS = np.array([(s, t) for s in NS for t in NT if (s, t) != (3, 5)], np.int32)     # 2500 x 3073 adds oracle time, no new case


@pytest.fixture(scope="module")
def scene():
    sc = synth.make_scene(7, 6500, 31, "dense")
    for v, n in {**NS, **NT}.items():
        sc.segs[v] = sc.segs[v][:n].copy()
    return sc


@pytest.fixture(scope="module")
def loaded(gpu_ctx, scene):
    gpu_ctx.set_views(util.scene_descs(scene), scene.segs)
    return gpu_ctx


def _fd(scene):
    return np.stack([synth.fundamental(scene.K[s], scene.R[s], scene.t[s], scene.K[t], scene.R[t], scene.t[t]).reshape(9) for s, t in PAIRS])


@pytest.mark.parametrize("knn", [10, -1])
def test_units_ref_gpu(loaded, scene, oracle, knn):
    """float semantics: the kNN best (knn 10) or every match (knn -1) of each row, as the oracle's restatement of the reference kernel"""
    loaded.match_pairs(PAIRS, util.pair_F(scene, PAIRS), 0.25, knn)
    total = 0
    for p, (s, t) in enumerate(PAIRS):
        pi = util.pair_inputs(scene, s, t)
        oc, oo, _, _ = oracle.match_lines(oracle.lib().orc_match_lines_f32, pi["ls"], pi["lt"], pi["F"], pi["Rs"], pi["Rt"], pi["Cs"], pi["Ct"],
                                          s, t, 0.25, max(knn, 0))
        counts, recs = loaded.pair_matches(p, len(pi["ls"]))
        assert np.array_equal(counts, oc), (s, t)
        f = ("tgt_seg", "overlap")
        assert util.rows_as_sets(counts, recs, f) == util.rows_as_sets(oc, oo, f), (s, t)
        if knn > 0:                                  # top-k rows come best first
            for r in range(len(counts)):
                ov = recs[r, :counts[r]]["overlap"]
                assert np.all(ov[:-1] >= ov[1:])
        total += int(oc.sum())
    assert total > 20000


@pytest.mark.parametrize("knn", [10, 0])
def test_units_ref_cpu(loaded, scene, oracle, knn):
    """double semantics: members, overlaps and depths bit for bit; keep-all rows also in the reference's ascending-target order"""
    Fd = _fd(scene)
    loaded.match_pairs_f64(PAIRS, Fd, 0.25, knn)
    RtKinv, C = synth.camera_blocks(scene)
    total = 0
    for p, (s, t) in enumerate(PAIRS):
        oc, oo, _, _ = oracle.match_lines(oracle.lib().orc_match_lines_f64, scene.segs[s], scene.segs[t], Fd[p], RtKinv[s].reshape(9),
                                          RtKinv[t].reshape(9), C[s], C[t], s, t, 0.25, knn, f64=True)
        counts, recs = loaded.pair_matches(p, len(scene.segs[s]))
        assert np.array_equal(counts, oc), (s, t)
        if knn > 0:
            assert util.rows_as_sets(counts, recs) == util.rows_as_sets(oc, oo), (s, t)
        else:
            for r in range(len(counts)):
                a, b = recs[r, :counts[r]], oo[r, :counts[r]]
                for f in ("tgt_seg", "overlap", "d_p1", "d_p2", "d_q1", "d_q2"):
                    assert a[f].tobytes() == b[f].tobytes(), (s, t, r, f)
        total += int(oc.sum())
    assert total > 20000


@pytest.mark.parametrize("knn", [10, -1])
def test_repeat_is_byte_identical(gpu_ctx, knn):
    """two identical calls on a scene of 3000-segment views (the benchmark's size) give the same counts and records, byte for byte"""
    sc = synth.make_scene(6, 3000, 1004, "ring2")
    pairs = synth.view_pairs(sc.neighbors)
    F = util.pair_F(sc, pairs)
    gpu_ctx.set_views(util.scene_descs(sc), sc.segs)
    runs = []
    for _ in range(2):
        gpu_ctx.match_pairs(pairs, F, 0.25, knn)
        counts, total = gpu_ctx.match_counts()
        runs.append((counts.copy(), total, [util.ordered_rows_sha(*gpu_ctx.pair_matches(p, 3000)).tobytes() for p in range(len(pairs))]))
    assert runs[0][1] > 10000
    assert runs[0][0].tobytes() == runs[1][0].tobytes() and runs[0][1] == runs[1][1]
    assert runs[0][2] == runs[1][2]
