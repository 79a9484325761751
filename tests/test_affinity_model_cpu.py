"""The CPU oracle's computingAffinityMatrix (OraclePipeline.affinity_raw / local2global) against the float64 sequential restatement
(tests/affinity_model.py), fed with the oracle's own kept matches, estimates, collinear lists and view parameters, on every scene
builder with the links off, at 2 px and at 5 px; and which paths of the loop each scene reaches.  The GPU side
(l3d_affinity_matrix / l3d_affinity_edges against the same model) is tests/test_affinity_paths_gpu.py.

Paths no scene can reach: a source-link pair lies within one view while direct and target-link pairs span two, so a source link
can only be rejected by another source link and a direct edge or target link never by a source link (asserted 0 below).
"Target link rejected by an earlier direct edge" needs kept lists that disagree: the link s -> w through s's target z is tried
only if the direct edge s -> z was new, and z ~ w, so s -> w can only have been taken by w's own direct edge w -> s while z did not
list s.  filterMatches drops a match below 10 % of its view's best score in one view and keeps its inverse in the other; at the
reference's 10 % that never happens on these scenes, at 30 % it does (test_stricter_filter_reaches_tlink_by_direct, and the GPU
test runs the device at 30 %)."""
import dataclasses
import functools

import numpy as np
import pytest

from tests import affinity_model as am

COLLIN = (-1.0, 2.0, 5.0)
TWO_SIGA_SQR, MIN_AFFINITY = 200.0, 0.5            # 2 * sigma_a^2 for sigma_a = 10 degrees; L3D_DEF_MIN_AFFINITY
RTOL = 1e-6                                        # measured: at most 1.9e-7 (float32 oracle against float64 model)
IMPOSSIBLE = ("direct_by_slink", "tlink_by_slink", "slink_by_direct", "slink_by_tlink")

# the paths each scene reaches with links on (2 px or 5 px), besides the depth branches every scene has
REACHES = {
    "whole_broken": ("direct_by_direct", "direct_by_tlink", "slink_by_slink", "tlink_skipped", "slink_gated", "slink_after_failed",
                     "id_by_tlink", "id_by_slink", "partner_no_estimate", "angle_gt_90"),
    "overlap": ("direct_by_direct", "direct_by_tlink", "slink_by_slink", "tlink_skipped", "slink_gated", "slink_after_failed",
                "id_by_tlink", "id_by_slink", "partner_no_estimate", "angle_gt_90"),
    "thirds": ("direct_by_direct", "direct_by_tlink", "tlink_by_tlink", "slink_by_slink", "tlink_skipped", "slink_gated",
               "slink_after_failed", "id_by_tlink", "id_by_slink", "partner_no_estimate", "angle_gt_90"),
}


def views_median(views):
    """med_scene_depth_lines as reconstruct3Dlines takes it: the median of the views' median depths above L3D_EPS"""
    d = sorted(md for _, md in views.values() if md > am.EPS)
    return d[len(d) // 2] if d else 0.0


@functools.lru_cache(maxsize=None)
def oracle_run(name, collin):
    """(pipeline, problem) after reconstruct3Dlines on the scene; the pipeline keeps affinity_raw and the scored lists"""
    from oracle import pyoracle as po
    sc = am.scene(name)
    P = po.OraclePipeline(False, True)
    P.add_scene(sc)
    P.match_images()
    assert P.reconstruct(3, False, collin) == 0
    cams = [int(c) for c in sc.cam_ids]
    views = {c: P.view_info(c) for c in cams}
    col = {c: P.collinear(c, len(sc.segs[i])) for i, c in enumerate(cams)} if collin > 0 else None
    best, pp = P.estimates()
    return P, am.problem(best, pp, [P.matches(c) for c in cams], col, views)


@pytest.mark.parametrize("collin", COLLIN)
@pytest.mark.parametrize("name", list(am.SCENES))
def test_oracle_matches_model(oracle, name, collin):
    P, pr = oracle_run(name, collin)
    r = am.restate(pr, TWO_SIGA_SQR, views_median(pr.views), MIN_AFFINITY)
    assert r.band == 0
    ei, ej, ew = P.affinity_raw()
    assert len(ei) > 5000
    assert np.array_equal(ei, r.ei) and np.array_equal(ej, r.ej)
    assert np.max(np.abs(ew - r.ew) / r.ew) <= RTOL
    assert [tuple(x) for x in P.local2global().tolist()] == r.l2g
    # the candidate list holds every accepted edge with its weight
    assert np.array_equal(np.array([r.cand[i][2] for i in r.acc.tolist()]), r.ew[0::2])


@pytest.mark.parametrize("name", list(am.SCENES))
def test_scene_reaches_its_paths(oracle, name):
    off = am.restate(oracle_run(name, -1.0)[1], TWO_SIGA_SQR, 4.0, MIN_AFFINITY)
    assert all(off.hits[p] == 0 for p in am.PATHS[1:15]) and off.chain == 2        # no links: only direct events, direct rejections
    hits, chain = {p: 0 for p in am.PATHS}, 0
    for collin in COLLIN[1:]:
        pr = oracle_run(name, collin)[1]
        r = am.restate(pr, TWO_SIGA_SQR, views_median(pr.views), MIN_AFFINITY)
        hits = {p: hits[p] + r.hits[p] for p in am.PATHS}
        chain = max(chain, r.chain)
    assert {p for p in REACHES[name] if hits[p] == 0} == set()
    assert all(hits[p] == 0 for p in IMPOSSIBLE)
    assert hits["depth_gt_cutoff"] > 0 and hits["depth_le_cutoff"] > 0
    assert chain >= 5


def refiltered(P, pr, perc):
    """pr with the kept lists filterMatches leaves at min_best_perc = perc, from the oracle's scored lists (scoring does not depend
    on the threshold, and an estimate's best match passes any threshold below 1)"""
    kept = {}
    for c in sorted(pr.views):
        m = P.scored(c)
        m = m[(m["score3D"] > 0) & (m["score3D"] > np.float32(perc) * m["score3D"].max(initial=0))]
        est = set(pr.est_seg[pr.est_cam == c].tolist())
        for ss, tc, ts in zip(m["src_seg"].tolist(), m["tgt_cam"].tolist(), m["tgt_seg"].tolist()):
            if ss in est:
                kept.setdefault((c, ss), []).append((tc, ts))
    return dataclasses.replace(pr, kept=kept)


def test_stricter_filter_reaches_tlink_by_direct(oracle):
    P, pr = oracle_run("thirds", 5.0)
    assert refiltered(P, pr, 0.1).kept == pr.kept                 # the refilter at the reference's 10 % is the oracle's filter
    r = am.restate(refiltered(P, pr, 0.3), TWO_SIGA_SQR, views_median(pr.views), MIN_AFFINITY)
    assert r.hits["tlink_by_direct"] > 0 and r.hits["tlink_by_tlink"] > 0 and r.band == 0


def test_similarity_edges():
    """similarity() on hand-made estimates: no estimate, a zero-length estimate, the NaN-ignoring fmin of a zero regulariser with
    a zero distance, and the cutoff dropped at med_scene_depth_lines = 0"""
    P = np.array([[0, 0, 4, 1, 0, 4], [0, 0, 4, 1, 0, 4], [0, 0, 4, 0, 0, 4], [1, 0, 4, 0, 0, 4.0]])
    pr = am.Problem(np.array([0, 1, 1, 2]), np.array([0, 0, 1, 0]), np.array([4.0, 0.0, 4.0, 4.0], np.float32),
                    np.array([4.0, 4.0, 4.0, 4.0], np.float32), P, {}, None, {0: (1e-3, 3.0), 1: (1e-3, 3.0), 2: (1e-3, 5.0)})
    s, f = am.similarities(pr, [0, 0, 0, 0], [-1, 1, 2, 3], 200.0, 0.0)
    assert s[0] == 0 and s[2] == 0                                   # no estimate; zero length
    assert s[1] == 1.0                                               # 0 / 0 on P1 (depth 0) is ignored by fmin, the rest is exp(0)
    assert s[3] == 1.0 and f["angle_gt_90"][3]                       # the reversed copy: 180 degrees folds to 0
    assert f["depth_gt_cutoff"][1] and f["depth_le_cutoff"][1]
    s5, _ = am.similarities(pr, [0], [3], 200.0, 2.0)                # a scene cutoff below the views' median depths
    assert s5[0] == 1.0
