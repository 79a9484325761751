"""The candidate model (tests/candidates_model.py) against the oracle matcher: with every target as a candidate it is the scan, for
both semantics and every kind of kNN; on hand-made rows it keeps ties, duplicates and empty lists as the matcher's rules say; and
feeding it to the oracle pipeline with full lists changes nothing downstream."""
import numpy as np
import pytest

from line3dpp_b200 import synth
from oracle import pyoracle
from tests import candidates_model as cm

KNNS = [1, 10, 32, 0, 40]


@pytest.fixture(scope="module")
def scene():
    return synth.make_scene(4, 300, 21, "ring2")


def _scan(scene, s, t, knn, f64):
    RtKinv, C = synth.camera_blocks(scene)
    F = synth.fundamental(scene.K[s], scene.R[s], scene.t[s], scene.K[t], scene.R[t], scene.t[t])
    fn = pyoracle.lib().orc_match_lines_f64 if f64 else pyoracle.lib().orc_match_lines_f32
    return pyoracle.match_lines(fn, scene.segs[s], scene.segs[t], F.reshape(9), RtKinv[s].reshape(9), RtKinv[t].reshape(9), C[s], C[t],
                                int(scene.cam_ids[s]), int(scene.cam_ids[t]), 0.25, knn, f64=f64, cap=None if knn > 0 else len(scene.segs[t]))[:2]


def _same_rows(a, b):
    (ca, ma), (cb, mb) = a, b
    assert np.array_equal(ca, cb)
    for r in range(len(ca)):
        assert ma[r, :ca[r]].tobytes() == mb[r, :cb[r]].tobytes(), r


@pytest.mark.parametrize("f64", [False, True])
@pytest.mark.parametrize("knn", KNNS)
@pytest.mark.parametrize("src,tgt", [(0, 1), (1, 0)])
def test_every_target_is_the_scan(scene, oracle, f64, knn, src, tgt):
    """every cell as a candidate (in either camera order of the pair, so both directions are sources) gives the matcher's rows"""
    keep = cm.pair_keep_all(scene, src, tgt, 0.25, f64)
    assert keep[0].sum() > 500
    Ns, Nt = len(scene.segs[src]), len(scene.segs[tgt])
    every = np.stack(np.meshgrid(np.arange(Ns), np.arange(Nt), indexing="ij"), -1).reshape(-1, 2)
    _same_rows(cm.restricted_rows(keep, every, knn), _scan(scene, src, tgt, knn, f64))
    _same_rows(cm.restricted_rows(keep, None, knn), _scan(scene, src, tgt, knn, f64))


def _rows(spec):
    """hand-made keep-all rows: spec = [[(tgt, overlap), ...] per row], ascending tgt"""
    cap = max(1, max(len(r) for r in spec))
    counts = np.array([len(r) for r in spec], np.int32)
    m = np.zeros((len(spec), cap), pyoracle.MATCH_DT)
    for i, row in enumerate(spec):
        for k, (t, ov) in enumerate(row):
            m[i, k]["src_seg"], m[i, k]["tgt_seg"], m[i, k]["overlap"], m[i, k]["d_p1"] = i, t, ov, t + 0.5
    return counts, m


def test_ties_duplicates_and_empty_lists():
    keep = _rows([[(0, 0.5), (3, 0.9), (5, 0.5), (7, 0.9), (9, 0.3)], [(1, 0.7), (2, 0.7)], []])
    cand = [(0, 9), (0, 7), (0, 5), (0, 5), (0, 0), (0, 7), (1, 4), (2, 1)]      # duplicates; row 1: a candidate that is no match
    c, m = cm.restricted_rows(keep, cand, 1)
    assert list(c) == [1, 0, 0] and m[0, 0]["tgt_seg"] == 7
    c, m = cm.restricted_rows(keep, cand, 10)
    assert list(c) == [4, 0, 0] and list(m[0, :4]["tgt_seg"]) == [7, 0, 5, 9]     # overlap descending, the smaller target on a tie
    c, m = cm.restricted_rows(keep, cand, 2)
    assert list(m[0, :2]["tgt_seg"]) == [7, 0]
    c, m = cm.restricted_rows(keep, cand, 0)
    assert list(c) == [4, 0, 0] and list(m[0, :4]["tgt_seg"]) == [0, 5, 7, 9]     # keep-all: ascending target
    c, m = cm.restricted_rows(keep, cand, 40)
    assert list(m[0, :4]["tgt_seg"]) == [7, 0, 5, 9]
    c, _ = cm.restricted_rows(keep, np.zeros((0, 2)), 10)                           # an empty list: no matches at all
    assert not c.any()
    c, m = cm.restricted_rows(keep, None, 32)
    assert list(c) == [5, 2, 0] and list(m[1, :2]["tgt_seg"]) == [1, 2]


def _pipeline(scene, source=None, knn=10):
    O = pyoracle.OraclePipeline(False, True, match_source=source)
    O.add_scene(scene)
    O.match_images(knn=knn)
    O.reconstruct(3, False)
    return O


@pytest.mark.parametrize("knn", [10, 0])
def test_oracle_pipeline_with_full_lists(oracle, knn):
    """OraclePipeline(match_source=model) with every cell of every pair listed: estimates, affinity, clusters and lines are the plain
    pipeline's"""
    sc = synth.make_scene(5, 150, 5, "ring2")
    plain = _pipeline(sc, knn=knn)
    lists = {}
    for a, b in plain.pairs():
        na, nb = len(sc.segs[list(sc.cam_ids).index(a)]), len(sc.segs[list(sc.cam_ids).index(b)])
        lists[(int(b), int(a))] = np.stack(np.meshgrid(np.arange(nb), np.arange(na), indexing="ij"), -1).reshape(-1, 2)   # reversed order
    model = _pipeline(sc, cm.match_source(sc, lists), knn=knn)
    assert np.array_equal(plain.pairs(), model.pairs())
    for cam in sc.cam_ids:
        assert plain.scored(cam).tobytes() == model.scored(cam).tobytes()
    (b0, p0), (b1, p1) = plain.estimates(), model.estimates()
    assert b0.tobytes() == b1.tobytes() and p0.tobytes() == p1.tobytes()
    for f in ("affinity_raw", "affinity", "local2global", "residuals", "segments3d"):
        a, b = getattr(plain, f)(), getattr(model, f)()
        a, b = (a if isinstance(a, tuple) else (a,)), (b if isinstance(b, tuple) else (b,))
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b)), f
    assert plain.num_lines() == model.num_lines() > 10
