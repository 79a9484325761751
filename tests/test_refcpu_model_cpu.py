"""The float64 model of the REF_CPU scoring sweep (tests/refcpu_model.py) against the oracle's own scoringCPU / filterMatches
restatement (oracle/l3d_oracle.cc) on the scenes the GPU tests use: outside the band every decision is the oracle's, every
score3D lies within the model's bound for the glibc build, and the closure's preconditions hold (one scene with U empty, one with
a similarity placed in band whose inverse entry U follows)."""
import numpy as np
import pytest

from line3dpp_b200 import synth
from tests import refcpu_model as rm
from tests import sweep_edges as E


def check_model_vs_oracle(res, scored, kept, est):
    """scores within E_cpu outside U, inside their interval in U; kept sets and best matches of the segments U does not reach
    are the model's"""
    best = {(int(b["src_cam"]), int(b["src_seg"])): (int(b["tgt_cam"]), int(b["tgt_seg"])) for b in est[0]}
    n = 0
    for cam, v in res.views.items():
        o = scored[cam]["score3D"].astype(np.float64)
        cert = ~v.uncertain
        assert (np.abs(o - v.score)[cert] <= v.E["cpu"][cert]).all(), cam
        assert ((o >= v.lo - v.slack) & (o <= v.hi + v.slack))[~cert].all(), cam
        ku = np.array(sorted(v.kept_u), np.int64)
        mine = scored[cam][v.kept & ~np.isin(v.seg, ku)]
        theirs = kept[cam][~np.isin(kept[cam]["src_seg"], ku)]
        for f in rm.IDS:
            assert np.array_equal(mine[f], theirs[f]), (cam, f)
        for sg, i in v.best_at.items():
            if sg not in v.kept_u and v.best_margin[sg] > 0:
                m = scored[cam][i]
                assert best[(cam, sg)] == (int(m["tgt_cam"]), int(m["tgt_seg"])), (cam, sg)
        n += int(cert.sum())
    return n


def test_ring3_model_vs_oracle_u_empty(oracle):
    """tests/test_refcpu_gpu.py's scene: U is empty, and the model reproduces the oracle's scores (most bit for bit)"""
    sc = synth.make_scene(8, 500, 31, "ring3")
    P = oracle.OraclePipeline(False, False)
    P.add_scene(sc)
    P.match_images()
    cams = rm.Cameras.of_scene(sc, [P.view_info(c)[0] for c in sc.cam_ids])
    res, scored, kept, est = rm.run_model(cams, P, sc.cam_ids, 200.0)
    assert res.size() == 0, res.events()
    assert check_model_vs_oracle(res, scored, kept, est) > 100000
    exact = sum(int((scored[c]["score3D"].astype(np.float64) == v.score).sum()) for c, v in res.views.items())
    assert exact > 0.99 * sum(len(m) for m in scored.values())
    # the band is a few ulps of 0.5 wide, not 1e-5
    W = rm.band_width(res)
    assert 0 < W < 16 * 2.0 ** -24, W


@pytest.mark.parametrize("name", ["sa10", "fixed"])
def test_sweep_edges_model_vs_oracle(oracle, name):
    """tests/test_sweep_edges_gpu.py::test_ref_cpu_vs_oracle's lists: on sa10 the placed similarity is in band, its entry's
    score sign is open and U reaches the target segment of its inverse entry"""
    from tests.test_sweep_edges_cpu import run_oracle
    sc = E.scene()
    params = E.PARAMS[name]
    L = E.build(sc, params, in_band=name == "sa10")
    O = run_oracle(oracle, L, params, False)
    cams = rm.Cameras.of_scene(sc, [O.view_info(c)[0] for c in sc.cam_ids])
    res, scored, kept, est = rm.run_model(cams, O, sc.cam_ids, 200.0)
    check_model_vs_oracle(res, scored, kept, est)
    ev = res.events()
    if name == "sa10":
        c = L.cases[-1]
        assert c.kind == "in_band" and abs(c.info["sim"] - 0.5) <= c.info["W"]
        v = res.views[c.view]
        i = np.flatnonzero((scored[c.view]["src_seg"] == c.seg) & (scored[c.view]["tgt_cam"] == c.tgt_cam))[0]
        assert v.in_band[i] and v.lo[i] == 0 < v.hi[i]                  # the sign of its score is open
        assert ev["sim"] == 1 and ev["inverse"] == 1
        assert c.tgt_seg in res.u_segments(c.tgt_cam)                   # ... and so is the target segment's list
    else:
        assert ev["sim"] == 0 and ev["inverse"] == 0
    assert res.size() <= 8, ev


def test_bound_arithmetic():
    """W of single similarities: exact inputs give exact outputs, and the angular term's bound grows with the libm ulps"""
    one = np.ones(1, np.float32)
    s, W = rm.sims(one, 0 * one, 0 * one, one, one, 200.0, np.zeros(1, bool))
    assert s[0] == 1.0 and W["gpu"][0] == 0.0 and W["cpu"][0] == 0.0      # expf(0) = 1, acosf(1) = 0
    dot = np.array([np.cos(np.radians(11.77))], np.float32)
    s, W = rm.sims(dot, 0 * one, 0 * one, one, one, 200.0, np.zeros(1, bool))
    assert abs(s[0] - 0.5) < 1e-2 and 0 < W["cpu"][0] < W["gpu"][0] < 64 * 2.0 ** -24
