"""k_match_topk's row slots at the kernel's geometry: a work unit of a pair whose target view takes several passes holds at most
MK_NSLOT = MK_WARPS * MK_SLOTS rows (256: 32 warps x 8 slots, l3d_match.cuh), one per slot.  Source views of MK_NSLOT - 1, MK_NSLOT and
MK_NSLOT + 1 rows fill every slot but one, every slot, and every slot plus a unit of one row; 2500 rows give several units of both
kinds.  Target views of 3072, 3073 and 6500 segments take one, two and three passes over the ring.  Every instantiation (REF_GPU /
REF_CPU semantics, top-k and keep-all) row by row against the CPU oracle."""
import numpy as np
import pytest

from line3dpp_b200 import synth
from tests import util

pytestmark = pytest.mark.gpu

NSLOT = 256
NS = {0: NSLOT - 1, 1: NSLOT, 2: NSLOT + 1, 3: 2500}
NT = {4: 3072, 5: 3073, 6: 6500}
PAIRS = np.array([(s, t) for s in NS for t in NT], np.int32)


@pytest.fixture(scope="module")
def scene():
    sc = synth.make_scene(7, 6500, 37, "dense")
    for v, n in {**NS, **NT}.items():
        sc.segs[v] = sc.segs[v][:n].copy()
    return sc


@pytest.fixture(scope="module")
def loaded(gpu_ctx, scene):
    gpu_ctx.set_views(util.scene_descs(scene), scene.segs)
    return gpu_ctx


@pytest.mark.parametrize("knn", [10, -1])
def test_slots_ref_gpu(loaded, scene, oracle, knn):
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


@pytest.mark.parametrize("knn", [10, -1])
def test_slots_ref_cpu(loaded, scene, oracle, knn):
    """double semantics: members, overlaps and depths bit for bit; keep-all rows also in the reference's ascending-target order"""
    Fd = np.stack([synth.fundamental(scene.K[s], scene.R[s], scene.t[s], scene.K[t], scene.R[t], scene.t[t]).reshape(9) for s, t in PAIRS])
    loaded.match_pairs_f64(PAIRS, Fd, 0.25, knn)
    RtKinv, C = synth.camera_blocks(scene)
    total = 0
    for p, (s, t) in enumerate(PAIRS):
        oc, oo, _, _ = oracle.match_lines(oracle.lib().orc_match_lines_f64, scene.segs[s], scene.segs[t], Fd[p], RtKinv[s].reshape(9),
                                          RtKinv[t].reshape(9), C[s], C[t], s, t, 0.25, max(knn, 0), f64=True)
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
