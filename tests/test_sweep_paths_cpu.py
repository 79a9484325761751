"""The oracle's restatement of the reference's host logic (OraclePipeline, REF_CPU semantics) pinned on the verbatim CPU reference
on W4 of tests/test_sweep_paths_gpu.py: 52 views with dense neighbours, segments matched into more than 48 target cameras.  The
GPU's REF_CPU sweep is checked against this restatement there, so this keeps that anchor honest above 48 cameras."""
import os

import numpy as np

from tests import util
from tests.test_ref_full_cpu import digest_matches
from tests.test_sweep_paths_gpu import CPU_GOLDEN, SC_MAP, WIDE, wide_scene


def test_oracle_host_logic_vs_verbatim_line3d_cc_wide(oracle):
    """every stage of the verbatim CPU reference on W4 (tests/golden/ref_full_wide_cpu_v1.npz, made by
    tests/golden/make_ref_wide_golden.py) against the restatement: scored lists (ids and geometry by digest, score sums to 1e-5),
    kept matches, regularisers, estimates, affinity edges, local ids, residuals and 3D segments"""
    z = np.load(CPU_GOLDEN)
    sc = wide_scene("w4")
    oracle.set_threads(os.cpu_count() or 1)
    O = oracle.OraclePipeline(False, 0)
    O.add_scene(sc)
    assert O.match_images(knn=WIDE["w4"][3]) == 0 and O.reconstruct(3, False) == 0
    oracle.set_threads(1)
    assert np.array_equal(z["pairs"], O.pairs())
    ncam = 0
    for cam in sc.cam_ids:
        m = O.scored(cam)
        assert len(m) == z[f"scored_n_{cam}"][0], f"scored {cam}"
        assert np.array_equal(digest_matches(m), z[f"scored_sha_{cam}"]), f"scored {cam}"
        assert abs(m["score3D"].astype(np.float64).sum() - z[f"scored_sum_{cam}"][0]) <= 1e-5 * max(1.0, abs(z[f"scored_sum_{cam}"][0]))
        k = O.matches(cam)
        assert len(k) == z[f"kept_n_{cam}"][0] and np.array_equal(digest_matches(k), z[f"kept_sha_{cam}"]), f"kept {cam}"
        assert abs(k["score3D"].astype(np.float64).sum() - z[f"kept_sum_{cam}"][0]) <= 1e-5 * max(1.0, abs(z[f"kept_sum_{cam}"][0]))
        assert tuple(z[f"view_info_{cam}"]) == tuple(np.float32(x) for x in O.view_info(cam))
        if cam < 4:
            ncam = max(ncam, max(len(np.unique(m["tgt_cam"][m["src_seg"] == s])) for s in np.unique(m["src_seg"])))
    assert ncam >= SC_MAP + 2, ncam          # the scene reaches past the GPU's 48-slot per-camera map
    bO, pO = O.estimates()
    assert len(bO) == z["est_n"][0] and np.array_equal(digest_matches(bO), z["est_sha"])
    np.testing.assert_allclose(pO[util.sample_idx(len(bO), len(z["est_P_sample"]))], z["est_P_sample"], rtol=0, atol=1e-13)
    ei, ej, ew = O.affinity_raw()
    assert len(ei) == z["aff_n"][0] > 1000 and np.array_equal(util.sha(ei, ej), z["aff_ij"])
    np.testing.assert_allclose(ew[util.sample_idx(len(ew), len(z["aff_w_sample"]))], z["aff_w_sample"], rtol=1e-6)
    assert np.array_equal(z["l2g"], O.local2global())
    assert z["num_lines"][0] == O.num_lines() > 100
    rR, rO = z["residuals"], O.residuals()
    assert all(np.array_equal(rR[f], rO[f]) for f in ("line", "cam", "seg"))
    sR, sO = z["segments3d"], O.segments3d()
    assert np.array_equal(sR["line"], sO["line"])
    np.testing.assert_allclose(sR["p1"], sO["p1"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(sR["p2"], sO["p2"], rtol=0, atol=1e-12)
