"""The hand-built lists of tests/sweep_edges.py on the oracle's CPU emulation (no GPU): the model places every case where it says,
and every band holds cases, so that tests/test_sweep_edges_gpu.py cannot pass without reaching them."""
import numpy as np
import pytest

from tests import sweep_edges as E

# cases every band must hold (orientation: on direct and on inverse entries each)
MIN_CASES = {"orientation": E.ORIENT_WANT, "similarity": 4, "tie": 5, "best_below_075": 3, "best_above_075": 3, "perc_below": 2,
             "perc_above": 2}
# the bands of angles at the cos_thr shortcut are reachable where the depth terms allow the rotation (see sweep_edges.PARAMS)
ANGLE_PARAMS = ("sa1", "fixed")


def check_populated(L, name):
    counts = E.band_counts(L)
    for band in list(E.ORIENT_BANDS) + list(E.SHORT_BANDS) + ["zero"]:
        for inverse in (False, True):
            assert counts.get((band, inverse), 0) >= MIN_CASES["orientation"], (name, band, inverse, counts)
    for band in list(E.SIM_BANDS) + (list(E.ANG_BANDS) if name in ANGLE_PARAMS else []):
        assert counts.get(band, 0) >= MIN_CASES["similarity"], (name, band, counts)
    for band in ("tie", "best_below_075", "best_above_075", "perc_below", "perc_above"):
        assert counts.get(band, 0) >= MIN_CASES[band], (name, band, counts)
    c = np.array([x.info["c"] for x in L.cases if x.band.startswith("bug_")])
    assert ((c > E.T2) & (c < E.OLD_C2 - 1e-9)).all()


def run_oracle(oracle, L, params, use_gpu, backend=None):
    P = oracle.OraclePipeline(False, use_gpu, backend=backend, match_source=L.source(oracle.MATCH_DT))
    P.add_scene(L.sc)
    assert P.match_images(knn=E.KNN, **params) == 0
    assert [tuple(p) for p in P.pairs()] == L.pairs
    return P


def outcome(P, cams):
    scored = {c: P.scored(c) for c in cams}
    kept = {c: P.matches(c) for c in cams}
    return scored, kept, P.estimates()[0]


@pytest.fixture(scope="module")
def sc():
    return E.scene()


@pytest.mark.parametrize("name", list(E.PARAMS))
def test_model_places_cases_as_the_oracle_decides(oracle, sc, name):
    """REF_GPU semantics with the CPU emulation of K_score_matches: every case's orientation, similarity and filter outcome is the
    model's, and view 7 has no positive score"""
    params = E.PARAMS[name]
    L = E.build(sc, params)
    check_populated(L, name)
    P = run_oracle(oracle, L, params, True)
    assert tuple(np.float32(x) for x in P.view_info(0))[0] == np.float32(L.geo.k[0])
    scored, kept, est = outcome(P, sc.cam_ids)
    bad = E.check_cases(L, scored, kept, est)
    assert not bad, sorted(set(b for b, _ in bad))
    last = scored[E.V - 1]
    assert len(last) > 0 and (last["score3D"] == 0).all() and len(kept[E.V - 1]) == 0


@pytest.mark.parametrize("name", ["sa10", "fixed"])
def test_model_orientation_vs_oracle_refcpu(oracle, sc, name):
    """REF_CPU semantics (scoringCPU restatement): the same orientation outcomes"""
    params = E.PARAMS[name]
    L = E.build(sc, params)
    P = run_oracle(oracle, L, params, False)
    scored, kept, est = outcome(P, sc.cam_ids)
    bad = [b for b, c in E.check_cases(L, scored, kept, est) if c.kind == "orientation"]
    assert not bad, sorted(set(bad))
