"""The scoring sweep (csrc/l3d_pipeline.cu) on the hand-built lists of tests/sweep_edges.py, which put its orientation, similarity
and filter decisions at their thresholds and at the edges of its shortcuts.  The lists reach the product through
Line3D::setShard's exchange (rank 0 of 2: the callback overwrites every row) and the oracle through orc_set_match_source.

  REF_GPU: every case's outcome is the model's (a failure names the bands), and every view's scored and kept lists, the
           estimates and the reconstruction are the oracle's on the verbatim reference kernels (ref_nofma)
  REF_CPU: the same orientation outcomes, kept matches and best matches as the oracle's scoringCPU restatement; scores at the
           libm / libdevice tolerance of tests/test_refcpu_gpu.py"""
import numpy as np
import pytest

from line3dpp_b200 import line3d
from tests import sweep_edges as E
from tests import util
from tests.test_sweep_edges_cpu import check_populated, outcome, run_oracle

pytestmark = pytest.mark.gpu


def run_product(L, params, use_gpu):
    """Line3D on the lists of L: rank 0 of 2, whose exchange callback replaces every row's count and records"""
    import torch
    from line3dpp_b200 import dist as l3dist
    counts, recs = L.buffers()
    calls = []

    def cb(_user, counts_dev, recs_dev, row_bounds, world, knn):
        try:
            rows = row_bounds[world]
            assert knn == E.KNN and rows == len(counts), (knn, rows, len(counts))
            l3dist.device_bytes(counts_dev, 4 * rows, 0).copy_(torch.from_numpy(counts.view(np.uint8)))
            l3dist.device_bytes(recs_dev, l3dist.REC_BYTES * knn * rows, 0).copy_(torch.from_numpy(recs.view(np.uint8).reshape(-1)))
            torch.cuda.synchronize()
            calls.append(knn)
            return 0
        except Exception as e:  # noqa: BLE001 - must not unwind through the C frame
            calls.append(e)
            return -1
    P = line3d.Line3D(neighbors_by_worldpoints=False, use_gpu=use_gpu)
    P.add_scene(L.sc)
    P._exchange_cb = l3dist._EXCHANGE_T(cb)
    P._chk(P.L.l3dpp_set_shard(P.h, 0, 2, P._exchange_cb, None), "setShard")
    P.match_images(knn=E.KNN, **params)
    assert calls == [E.KNN], calls
    assert [tuple(p) for p in P.pairs()] == L.pairs
    for cam in L.sc.cam_ids:
        assert np.float32(P.view_info(cam)[0]) == np.float32(L.geo.k[cam]), cam
    return P


@pytest.fixture(scope="module")
def sc():
    return E.scene()


@pytest.fixture(scope="module")
def ref_gpu_runs(oracle, ref_nofma, sc):
    """per parameter set: the lists, the product (REF_GPU) and the oracle on the verbatim reference kernels, both reconstructed"""
    runs = {}
    for name, params in E.PARAMS.items():
        L = E.build(sc, params)
        P = run_product(L, params, True)
        O = run_oracle(oracle, L, params, True, backend=ref_nofma)
        runs[name] = (L, P, O)
    yield runs
    for _, P, _ in runs.values():
        P.close()


def product_outcome(P, cams):
    return {c: P.view_matches(c, False) for c in cams}, {c: P.view_matches(c, True) for c in cams}, P.estimates()[0]


@pytest.mark.parametrize("name", list(E.PARAMS))
def test_ref_gpu_case_outcomes(ref_gpu_runs, name):
    L, P, _ = ref_gpu_runs[name]
    check_populated(L, name)
    scored, kept, est = product_outcome(P, L.sc.cam_ids)
    bad = E.check_cases(L, scored, kept, est)
    assert not bad, "cases decided against the model in bands " + ", ".join(sorted(set(b for b, _ in bad))) + \
        (" (bug_*: the band (cos T2, c2 - 1e-9) the double shortcut dropped)" if any(b.startswith("bug_") for b, _ in bad) else "")
    last = scored[E.V - 1]
    assert len(last) > 0 and (last["score3D"] == 0).all() and len(kept[E.V - 1]) == 0


@pytest.mark.parametrize("name", list(E.PARAMS))
def test_ref_gpu_vs_verbatim_kernels(ref_gpu_runs, name):
    """scored and kept lists bit for bit (order, ids, depths, score3D), estimates (best records exactly, P to 1e-12), then the
    reconstruction (util.check_reconstruction)"""
    L, P, O = ref_gpu_runs[name]
    n = 0
    for cam in L.sc.cam_ids:
        g, o = P.view_matches(cam, False), O.scored(cam)
        assert len(g) == len(o) and np.array_equal(util.match_sha(g), util.match_sha(o)), f"scored list of view {cam}"
        assert np.array_equal(util.match_sha(P.view_matches(cam, True)), util.match_sha(O.matches(cam))), f"kept list of view {cam}"
        n += len(g)
    bP, pP = P.estimates()
    bO, pO = O.estimates()
    assert len(bP) == len(bO) > 100 and np.array_equal(util.match_sha(bP), util.match_sha(bO))
    np.testing.assert_allclose(pP, pO, rtol=0, atol=1e-12)
    P.reconstruct_3d_lines(3, False)
    assert O.reconstruct(3, False) == 0
    rec = util.reconstruction_record(O.local2global(), O.affinity_raw(), O.affinity(), O.num_lines(), O.residuals(), O.segments3d())
    st = P.stats()
    assert st["lines3D"] > 10, st["lines3D"]
    util.check_reconstruction(rec, "", P.local2global(), P.affinity(raw=True), P.affinity(raw=False), st["lines3D"], P.residuals(),
                              P.segments3d(), 1e-6)


@pytest.mark.parametrize("name", ["sa10", "fixed"])
def test_ref_cpu_vs_oracle(oracle, sc, name):
    """REF_CPU: list membership (the orientation outcomes), kept matches and best matches as the oracle's; scores within the
    libm / libdevice tolerance, and a score outside it only where a similarity lies within that tolerance of sim_t (counted)"""
    params = E.PARAMS[name]
    L = E.build(sc, params)
    P = run_product(L, params, False)
    O = run_oracle(oracle, L, params, False)
    near = 0
    for cam in sc.cam_ids:
        g, o = P.view_matches(cam, False), O.scored(cam)
        assert len(g) == len(o), cam
        for f in ("src_seg", "tgt_cam", "tgt_seg", "d_p1", "d_p2", "d_q1", "d_q2"):
            assert np.array_equal(util.bits(g[f]) if g.dtype[f].kind == "f" else g[f], util.bits(o[f]) if o.dtype[f].kind == "f" else o[f]), (cam, f)
        bad = ~np.isclose(g["score3D"], o["score3D"], rtol=1e-5, atol=1e-6)     # TOLERANCE: libm vs libdevice expf/acosf
        d = np.abs(g["score3D"][bad].astype(np.float64) - o["score3D"][bad].astype(np.float64))
        assert (np.abs(d - E.SIM_T * np.maximum(np.round(d / E.SIM_T), 1)) <= 1e-4).all(), (cam, d[:8])
        near += int(bad.sum())
        if not bad.any():
            kg, ko = P.view_matches(cam, True), O.matches(cam)
            for f in ("src_seg", "tgt_cam", "tgt_seg"):
                assert np.array_equal(kg[f], ko[f]), (cam, f)
    assert near <= 3, near
    bP, bO = P.estimates()[0], O.estimates()[0]
    assert len(bP) == len(bO)
    for f in ("src_cam", "src_seg", "tgt_cam", "tgt_seg"):
        assert np.array_equal(bP[f], bO[f]), f
    scored, kept, est = product_outcome(P, sc.cam_ids)
    bad = [b for b, c in E.check_cases(L, scored, kept, est) if c.kind == "orientation"]
    assert not bad, sorted(set(bad))
    P.close()
