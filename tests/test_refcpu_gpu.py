"""REF_CPU semantics on the GPU (SURVEY.md §8(b) dual-semantics switch; rows a3 / a7): the reference's CPU twins
matchingCPU (line3D.cc:900-1015) and scoringCPU (1208-1294) computed by the GPU, checked against the CPU oracle's
restatement of them (oracle/l3d_oracle.cc: orc_match_lines_f64, scoring_cpu).  The matching part uses IEEE double
add/mul/div/sqrt only and is compared BIT FOR BIT; scoring goes through expf/acosf, whose CUDA and glibc versions differ by
ulps: every difference is accounted for by the float64 model of tests/refcpu_model.py (scores within its per-entry bound, no
decision near a threshold on this scene)."""
import numpy as np
import pytest

from line3dpp_b200 import line3d, synth
from tests import util

pytestmark = pytest.mark.gpu


def _pair_inputs_f64(scene, s, t):
    RtKinv, C = synth.camera_blocks(scene)
    F = synth.fundamental(scene.K[s], scene.R[s], scene.t[s], scene.K[t], scene.R[t], scene.t[t])
    return dict(ls=scene.segs[s], lt=scene.segs[t], F=F.reshape(9), Rs=RtKinv[s].reshape(9), Rt=RtKinv[t].reshape(9), Cs=C[s], Ct=C[t])


@pytest.mark.parametrize("knn", [10, 3])
def test_f64_topk_bit_exact_vs_oracle(gpu_ctx, oracle, knn):
    scene = synth.make_scene(6, 900, 21, "ring2")
    pairs = synth.view_pairs(scene.neighbors)
    Fd = np.stack([synth.fundamental(scene.K[s], scene.R[s], scene.t[s], scene.K[t], scene.R[t], scene.t[t]).reshape(9) for s, t in pairs])
    gpu_ctx.set_views(util.scene_descs(scene), scene.segs)
    gpu_ctx.match_pairs_f64(pairs, Fd, 0.25, knn)
    assert gpu_ctx.L.l3d_match_semantics(gpu_ctx.h) == 1
    n_total = 0
    for pi, (s, t) in enumerate(pairs):
        inp = _pair_inputs_f64(scene, s, t)
        oc, om, ototal, _ = oracle.match_lines(oracle.lib().orc_match_lines_f64, inp["ls"], inp["lt"], inp["F"], inp["Rs"], inp["Rt"],
                                               inp["Cs"], inp["Ct"], scene.cam_ids[s], scene.cam_ids[t], 0.25, knn, f64=True)
        gc, gr = gpu_ctx.pair_matches(pi, len(inp["ls"]))
        assert np.array_equal(gc, oc), f"pair {pi}: per-row match counts differ"
        assert util.rows_as_sets(gc, gr) == util.rows_as_sets(oc, om), f"pair {pi}: kNN members / overlaps / depths differ"
        n_total += int(oc.sum())
    assert n_total > 2000


def test_f64_differs_from_f32_semantics(gpu_ctx):
    """the two semantics are different functions (SURVEY §8a divergences 1, 4): make sure the switch switches something"""
    scene = synth.make_scene(4, 1200, 22, "ring1")
    pairs = synth.view_pairs(scene.neighbors)
    Fd = np.stack([synth.fundamental(scene.K[s], scene.R[s], scene.t[s], scene.K[t], scene.R[t], scene.t[t]).reshape(9) for s, t in pairs])
    gpu_ctx.set_views(util.scene_descs(scene), scene.segs)
    gpu_ctx.match_pairs_f64(pairs, Fd, 0.25, 10)
    c64, r64 = gpu_ctx.pair_matches(0, len(scene.segs[pairs[0][0]]))
    gpu_ctx.match_pairs(pairs, Fd.astype(np.float32), 0.25, 10)
    assert gpu_ctx.L.l3d_match_semantics(gpu_ctx.h) == 0
    c32, r32 = gpu_ctx.pair_matches(0, len(scene.segs[pairs[0][0]]))
    same_members = sum(sorted(r64[r, :c64[r]]["tgt_seg"]) == sorted(r32[r, :c32[r]]["tgt_seg"]) for r in range(len(c64)))
    assert same_members > 0.97 * len(c64)                       # same geometry ...
    assert util.rows_as_sets(c64, r64) != util.rows_as_sets(c32, r32)   # ... different arithmetic


@pytest.fixture(scope="module")
def scene():
    return synth.make_scene(8, 500, 31, "ring3")


def test_refcpu_pipeline_vs_oracle(scene, oracle):
    """every difference accounted for (tests/refcpu_model.py): on this scene no similarity lies within the libm band of 0.5 and
    no keep / best decision within the score bound, so U is empty and everything is exact - lists and their order, depths,
    score3D within the per-entry bound E (a few ulps), kept sets, best matches, estimates bit for bit, the reconstruction's line
    count (its affinity weights: see below)"""
    from tests import refcpu_model as rm
    L = line3d.Line3D(neighbors_by_worldpoints=False, use_gpu=False)
    L.add_scene(scene)
    L.match_images()
    P = oracle.OraclePipeline(False, False)          # use_gpu = False: matchingCPU + scoringCPU
    P.add_scene(scene)
    P.match_images()
    cams = rm.Cameras.of_scene(scene, [P.view_info(c)[0] for c in scene.cam_ids])
    res, scored, kept, est = rm.run_model(cams, P, scene.cam_ids, 200.0)
    assert res.size() == 0, res.events()              # precondition: the scene where everything is exact
    st = rm.check_run(res, scored, kept, est, lambda c: L.view_matches(c, False), lambda c: L.view_matches(c, True), L.estimates())
    print("REF_CPU ring3: |U| = 0,", st)
    assert st["entries"] > 5000 and st["est"] > 1000, st
    # reconstruction: no diffusion in REF_CPU (line3D.cc:1729).  Kept matches and estimates are identical, so the affinity
    # matrix is built from identical inputs; its weights go through expf (libdevice vs glibc) and could flip only within a few
    # ulps of min_affinity - tests/affinity_model.py counts none on this scene (asserted), so the line counts are equal.
    from tests import affinity_model as am
    from tests.test_affinity_model_cpu import views_median
    views = {int(c): P.view_info(c) for c in scene.cam_ids}
    best, pp = P.estimates()
    pr = am.problem(best, pp, [P.matches(c) for c in scene.cam_ids], None, views)
    L.reconstruct_3d_lines(3, True)
    assert P.reconstruct(3, True) == 0
    assert am.restate(pr, 200.0, views_median(pr.views), 0.5).band == 0
    nl, no = L.stats()["lines3D"], P.num_lines()
    assert no > 100 and nl == no, (nl, no)
    L.close()
