"""k_match_topk on target views that take two passes over the resident level-1 ring (3 stages x 512 entries = 1536 targets): every
instantiation (REF_GPU / REF_CPU semantics, top-k and keep-all) row by row against the CPU oracle.  Target sizes: 1537 (the second
pass holds one entry), 2048 (the second pass is exactly one full stage) and 3000 (the benchmark's view size)."""
import numpy as np
import pytest

from line3dpp_b200 import synth
from tests import util

pytestmark = pytest.mark.gpu

NT = {1: 3000, 2: 1537, 3: 2048}
PAIRS = np.array([(0, 1), (0, 2), (0, 3)], np.int32)


@pytest.fixture(scope="module")
def scene():
    sc = synth.make_scene(4, 3000, 29, "dense")
    sc.segs[0] = sc.segs[0][:300].copy()                # 300 source rows: five CTAs per pair, the last one partial
    for v, n in NT.items():
        sc.segs[v] = sc.segs[v][:n].copy()
    return sc


@pytest.fixture(scope="module")
def loaded(gpu_ctx, scene):
    gpu_ctx.set_views(util.scene_descs(scene), scene.segs)
    return gpu_ctx


def _fd(scene):
    return np.stack([synth.fundamental(scene.K[s], scene.R[s], scene.t[s], scene.K[t], scene.R[t], scene.t[t]).reshape(9) for s, t in PAIRS])


@pytest.mark.parametrize("knn", [10, -1])
def test_two_pass_targets_ref_gpu(loaded, scene, oracle, knn):
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
    assert total > 3000


@pytest.mark.parametrize("knn", [10, 0])
def test_two_pass_targets_ref_cpu(loaded, scene, oracle, knn):
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
    assert total > 3000
