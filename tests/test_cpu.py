"""CPU-only tests (`pytest -m "not gpu"`): the oracle against the golden vectors produced by the UNMODIFIED reference
kernels on the GPU (tests/golden/), against the reference's clustering.cc compiled in place (runs on the CPU), the
oracle pipeline on synthetic scenes with known 3D lines, host-side sharding logic, and the C-ABI surface of the product
library (load + exported symbols; no compute without a GPU)."""
import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from line3dpp_b200 import synth
from tests import util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_kernels_v1.npz")


@pytest.fixture(scope="module")
def gold():
    if not os.path.exists(GOLD):
        pytest.skip("golden vectors not generated yet (tests/golden/make_golden.py on a GPU box)")
    return np.load(GOLD)


@pytest.fixture(scope="module")
def gscene(gold):
    v, n, seed = [int(x) for x in gold["scene_args"]]
    sc = synth.make_scene(v, n, seed, "dense")
    assert np.array_equal(np.stack(sc.segs), gold["segs"]), "synthetic scene generator changed: regenerate the golden file"
    return sc


# ---------------------------------------------------------------------------------------------- oracle vs golden
@pytest.mark.parametrize("tag,s,t", [("p01", 0, 1), ("p24", 2, 4)])
def test_oracle_match_dense_vs_reference_golden(oracle, gold, gscene, tag, s, t):
    g = lambda k: gold[f"{tag}_{k}"]
    dep, ov, _ = oracle.match_dense(oracle.lib().orc_match_dense_f32, gscene.segs[s], gscene.segs[t], g("F"), g("Rs"), g("Rt"), g("Cs"), g("Ct"), 0.25)
    assert np.array_equal(util.bits(ov), util.bits(g("dense_ov")))            # overlap: bit-exact on the CPU
    sel = g("dense_ov") > 0.25
    assert sel.sum() > 200
    rel = np.abs(dep[sel] - g("dense_dep")[sel]) / np.maximum(np.abs(g("dense_dep")[sel]), 1e-3)
    assert np.median(rel) < 1e-6 and np.quantile(rel, 0.999) < 1e-2          # depths: host rsqrt vs MUFU.RSQ
    assert np.array_equal(dep[~sel], g("dense_dep")[~sel])                   # -1 everywhere else


@pytest.mark.parametrize("tag,s,t", [("p01", 0, 1), ("p24", 2, 4)])
def test_oracle_knn_lists_vs_reference_golden(oracle, gold, gscene, tag, s, t):
    g = lambda k: gold[f"{tag}_{k}"]
    counts, out, total, _ = oracle.match_lines(oracle.lib().orc_match_lines_f32, gscene.segs[s], gscene.segs[t], g("F"), g("Rs"), g("Rt"), g("Cs"), g("Ct"), s, t, 0.25, 10)
    assert np.array_equal(counts, g("knn_counts")) and total == g("knn_counts").sum()
    ref = g("knn")
    for r in range(len(counts)):
        a, b = out[r, :counts[r]], ref[r, :counts[r]]
        assert np.array_equal(a["tgt_seg"], b["tgt_seg"]) and np.array_equal(util.bits(a["overlap"]), util.bits(b["overlap"]))


def test_oracle_scores_vs_reference_golden(oracle, gold, gscene):
    p = gold["score_params"]
    scores, _ = oracle.score_matches(oracle.lib().orc_score_matches_f32, gscene.segs[0], gold["score_m4"], gold["score_ranges"], gold["score_reg"],
                                     gold["score_R"], gold["score_C"], float(p[0]), float(p[1]), float(p[2]))
    ref = gold["score_out"]
    assert len(ref) > 1000 and (ref > 0).sum() > 100
    off = ~np.isclose(scores, ref, rtol=1e-4, atol=1e-5)
    assert off.mean() < 5e-3       # a similarity at the 0.5 truncation may flip with a 1-ulp expf/acosf difference
    assert np.median(np.abs(scores - ref)) < 1e-6


def test_oracle_rdd_vs_reference_golden(oracle, gold):
    n = int(gold["rdd_n"][0])
    oi, oj, ow, _ = oracle.rdd(oracle.lib().orc_rdd_f32, gold["rdd_ei"], gold["rdd_ej"], gold["rdd_ew"], n)
    assert np.array_equal(oi, gold["rdd_oi"]) and np.array_equal(oj, gold["rdd_oj"])
    assert np.array_equal(util.bits(ow), util.bits(gold["rdd_ow"]))           # + - * / only: bit-exact


def test_oracle_cluster_vs_reference_golden(oracle, gold):
    n = int(gold["rdd_n"][0])
    lab = oracle.cluster(oracle.lib().orc_cluster, gold["rdd_ei"], gold["rdd_ej"], gold["rdd_ew"], n)
    assert np.array_equal(lab, gold["cluster_labels"])
    lab2 = oracle.cluster(oracle.lib().orc_cluster, gold["rdd_oi"], gold["rdd_oj"], gold["rdd_ow"], n)
    assert np.array_equal(lab2, gold["cluster_labels_rdd"])


def test_oracle_cluster_vs_reference_clustering_cc_live(oracle):
    """the reference's clustering.cc (compiled in place into oracle/_ref, tests/golden/make_ref_cpu_golden.py) on random graphs:
    its labels are stored in tests/golden/ref_cluster_live_v1.npz"""
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from make_ref_cpu_golden import cluster_graphs
    g = np.load(os.path.join(ROOT, "tests", "golden", "ref_cluster_live_v1.npz"))
    for k, (n, ei, ej, ew) in enumerate(cluster_graphs()):
        a = oracle.cluster(oracle.lib().orc_cluster, ei, ej, ew, n)
        assert np.array_equal(a, g[f"labels_{k}"])


# ---------------------------------------------------------------------------------------------- oracle pipeline sanity
def _dist_to_gt(pts, gt):
    a = gt[:, :3]
    d = gt[:, 3:] - a
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    w = pts[:, None, :] - a[None]
    return np.linalg.norm(w - (w * d[None]).sum(-1, keepdims=True) * d[None], axis=-1).min(1)


@pytest.mark.parametrize("use_gpu,diffusion", [(1, False), (1, True), (0, False)])
def test_oracle_pipeline_recovers_ground_truth_lines(oracle, use_gpu, diffusion):
    sc = synth.make_scene(10, 250, 9, "ring3")
    P = oracle.OraclePipeline(False, use_gpu)
    P.add_scene(sc)
    assert P.match_images() == 0
    assert P.pair_evals() == sum(len(sc.segs[s]) * len(sc.segs[t]) for s, t in synth.view_pairs(sc.neighbors))
    assert np.array_equal(P.pairs(), synth.view_pairs(sc.neighbors))
    assert P.reconstruct(3, diffusion) == 0
    s = P.segments3d()
    assert P.num_lines() > 150
    assert np.median(_dist_to_gt(s["p1"], sc.lines3d)) < 5e-3 and np.median(_dist_to_gt(s["p2"], sc.lines3d)) < 5e-3


def test_oracle_gpu_and_cpu_semantics_agree_statistically(oracle):
    sc = synth.make_scene(10, 250, 9, "ring3")
    n = []
    for use_gpu in (1, 0):
        P = oracle.OraclePipeline(False, use_gpu)
        P.add_scene(sc)
        P.match_images()
        P.reconstruct(3, False)
        n.append(P.num_lines())
    assert abs(n[0] - n[1]) <= 0.05 * n[0]


def test_oracle_edge_cases(oracle):
    L = oracle.lib()
    P = oracle.OraclePipeline(False, 1)
    K = np.array([[1000., 0, 500], [0, 1000., 400], [0, 0, 1]])
    seg = np.array([[10, 10, 100, 100]], np.float32)
    assert P.add_view(0, 600, 400, K, np.eye(3), np.zeros(3), 1.0, [1], seg) == -1     # image too small (line3D.cc:119)
    assert P.add_view(0, 1000, 800, K, np.eye(3), np.zeros(3), 1.0, [], seg) == -3      # no neighbours (line3D.cc:154)
    assert P.add_view(0, 1000, 800, K, np.eye(3), np.zeros(3), 1.0, [1], seg) == 0
    assert P.add_view(0, 1000, 800, K, np.eye(3), np.zeros(3), 1.0, [1], seg) == -2     # duplicate id (line3D.cc:130)
    assert P.match_images() == 0                                                        # neighbour 1 does not exist: nothing to match
    assert P.reconstruct(3, False) == -1                                                # no estimates (line3D.cc:1712)
    # degenerate geometry: identical cameras -> F = 0 -> every intersection invalid -> no matches, no crash
    z = np.zeros(9, np.float32)
    c, o, tot, _ = oracle.match_lines(L.orc_match_lines_f32, seg, seg, z, np.eye(3, dtype=np.float32).ravel(), np.eye(3, dtype=np.float32).ravel(),
                                      np.zeros(3, np.float32), np.zeros(3, np.float32), 0, 1, 0.25, 10)
    assert tot == 0


# ---------------------------------------------------------------------------------------------- host logic
def test_view_pairs_follow_reference_order():
    nb = [np.array([1, 2], np.uint32), np.array([0], np.uint32), np.array([3], np.uint32), np.array([0, 2], np.uint32)]
    assert synth.view_pairs(nb).tolist() == [[0, 1], [0, 2], [2, 3], [3, 0]]
    assert len(synth.view_pairs(synth.ring_neighbors(1000, 5))) == 5000
    assert len(synth.view_pairs(synth.dense_neighbors(200))) == 19900


def test_scene_shards_are_consistent():
    full = synth.make_scene(12, 100, 4, "ring2")
    part = synth.make_scene_views(12, 100, 4, "ring2", [3, 4, 5])
    for v in (3, 4, 5):
        assert np.array_equal(full.segs[v], part.segs[v])
    assert len(part.segs[0]) == 0 and np.array_equal(full.K, part.K) and np.array_equal(full.R, part.R)



# ---------------------------------------------------------------------------------------------- collinearity (SURVEY §8f-3)
GOLD_COLLIN = os.path.join(ROOT, "tests", "golden", "ref_collinear_v1.npz")


@pytest.mark.parametrize("name", ["v0", "v2", "edge"])
def test_oracle_collinear_vs_reference_golden(oracle, name):
    """orc_collinear_f32 == the UNMODIFIED K_collinearity run on the GPU (tests/golden/make_golden_collinear.py)"""
    if not os.path.exists(GOLD_COLLIN):
        pytest.skip("collinearity golden vectors not generated yet (tests/golden/make_golden_collinear.py on a GPU box)")
    g = np.load(GOLD_COLLIN)
    segs = g[f"{name}_segs"]
    if name != "edge":
        v, n, seed = [int(x) for x in g["scene_args"]]
        sc = synth.make_scene(v, n, seed, "ring1", collinear=True)
        assert np.array_equal(sc.segs[int(name[1:])], segs), "synthetic scene generator changed: regenerate the golden file"
    for t in (0.5, 2.0, 6.0):
        Cm, _ = oracle.collinear(oracle.lib().orc_collinear_f32, segs, t)
        assert np.array_equal(np.argwhere(Cm == 1).astype(np.int32), g[f"{name}_t{t}"]), (name, t)


def test_oracle_collinear_properties(oracle):
    """symmetric, empty diagonal, monotone in the threshold, float and double paths agree on well-conditioned input,
    and the fragments of a broken 3D line are found"""
    sc = synth.make_scene(4, 300, 95, "ring1", collinear=True)
    L = oracle.lib()
    prev = None
    for t in (1.0, 2.0, 5.0):
        a, _ = oracle.collinear(L.orc_collinear_f32, sc.segs[1], t)
        b, _ = oracle.collinear(L.orc_collinear_f64, sc.segs[1], t)
        assert np.array_equal(a, a.T) and not a.diagonal().any() and np.array_equal(a, b)
        if prev is not None:
            assert np.all(a >= prev)
        prev = a
    ids = sc.line_ids[1]
    frag = {(i, j) for i in range(len(ids)) for j in range(len(ids)) if i != j and ids[i] // 2 == ids[j] // 2}
    found = {tuple(x) for x in np.argwhere(prev == 1)}
    assert len(frag) > 20 and len(frag & found) >= 0.9 * len(frag)
    e, _ = oracle.collinear(L.orc_collinear_f32, np.zeros((0, 4), np.float32), 2.0)
    assert e.shape == (0, 0)


@pytest.mark.parametrize("use_gpu", [1, 0])
def test_oracle_collinearity_links_merge_fragments(oracle, use_gpu):
    sc = synth.make_scene(8, 300, 3, "ring2", collinear=True)
    out = {}
    for ct in (-1.0, 2.0):
        P = oracle.OraclePipeline(False, use_gpu)
        P.add_scene(sc)
        P.match_images()
        assert P.reconstruct(3, bool(use_gpu), ct) == 0
        out[ct] = (P.num_lines(), len(P.affinity_raw()[0]), sum(len(P.collinear(c, len(s))[1]) for c, s in zip(sc.cam_ids, sc.segs)))
        s = P.segments3d()
        assert np.median(_dist_to_gt(s["p1"], sc.lines3d)) < 5e-3
    assert out[-1.0][2] == 0 and out[2.0][2] > 300
    assert out[2.0][1] > out[-1.0][1] and out[2.0][0] < out[-1.0][0]


# ---------------------------------------------------------------------------------------------- line bundling (SURVEY §8f-4)
def _np_cost(x, cams, rc, xy):
    """independent numpy restatement of the bundling cost of ONE line (optimization.h:66-162 + HuberLoss(2)), no derivatives"""
    om, s = x[0], x[1:]
    nm = s @ s
    sx = np.array([[0, -s[2], s[1]], [s[2], 0, -s[0]], [-s[1], s[0], 0]])
    Q = ((1 - nm) * np.eye(3) + 2 * sx + 2 * np.outer(s, s)) / (1 + nm)
    l, m = Q[:, 0], om * Q[:, 1]
    c = 0.0
    for cam, o in zip(rc, xy):
        R, C, fx, fy, px, py = cams[cam, :9].reshape(3, 3), cams[cam, 9:12], *cams[cam, 12:16]
        q = R @ (m - np.cross(C, l))
        pl = np.array([fy * q[0], fx * q[1], -fy * px * q[0] - fx * py * q[1] + fx * fy * q[2]])
        d = np.hypot(pl[0], pl[1])
        dr = (o[2:] - o[:2]) / np.linalg.norm(o[2:] - o[:2])
        ang = np.arccos(np.clip((pl[0] * -dr[1] + pl[1] * dr[0]) / d, -1, 1))
        ang = min(ang, np.pi - ang)
        r = np.array([pl[0] * o[0] + pl[1] * o[1] + pl[2], pl[0] * o[2] + pl[1] * o[3] + pl[2]]) / d * np.exp(2 * ang)
        sq = r @ r
        c += 0.5 * (sq if sq <= 4 else 4 * np.sqrt(sq) - 4)
    return c


def test_oracle_optimizer_vs_reference_ceres_fixture(oracle):
    """orc_optimize_lines from the reference's UNOPTIMISED result lines + residuals reproduces the reference's own
    OPTIMIZED result (testdata/Line3D++_ref, both files; 2489 clusters with identical residual sets).  The fixture text has
    ~5e-6 of rounding; LineOptimizer moves the lines by 3.8e-4 (median), up to 1.6e-2."""
    from tests import nvm_util as nu
    before, after, ptr, res = nu.load_opt_pairs()
    cams, shift = nu.optimizer_inputs(nu.load_inputs())
    b = before + np.tile(shift, 2)
    out, valid, summ = oracle.optimize_lines(oracle.lib().orc_optimize_lines, b, ptr, res[:, 0].astype(np.int32), res[:, 2:6], cams, 250)
    out -= np.tile(shift, 2)
    assert valid.all() and summ[3] == 0 and summ[5] == len(before)              # converged, every line free
    assert summ[2] < 0.85 * summ[1]                                             # total cost 9514 -> ~7950
    moved, gap = nu.line_gap(after, before), nu.line_gap(after, out)
    assert np.median(moved) > 3e-4
    assert np.median(gap) < 2.5e-5 and np.percentile(gap, 90) < 1.5e-4 and np.percentile(gap, 99) < 8e-4, (np.median(gap), np.percentile(gap, [90, 99]))
    big = moved > 1e-3                                                           # where the reference really moved a line we follow it
    assert big.sum() > 200 and np.median(gap[big] / moved[big]) < 0.05


def test_oracle_optimizer_reaches_a_minimum_of_the_independent_cost(oracle):
    """the final Cayley parameters minimise an INDEPENDENT numpy restatement of the robust cost: scipy cannot improve them"""
    from scipy.optimize import minimize
    from tests import nvm_util as nu
    before, after, ptr, res = nu.load_opt_pairs()
    cams, shift = nu.optimizer_inputs(nu.load_inputs())
    sel = np.arange(0, 600, 20)
    b = (before + np.tile(shift, 2))[sel]
    p2 = np.concatenate([[0], np.cumsum(np.diff(ptr)[sel])])
    rr = np.concatenate([res[ptr[i]:ptr[i + 1]] for i in sel])
    out, valid, summ = oracle.optimize_lines(oracle.lib().orc_optimize_lines, b, p2, rr[:, 0].astype(np.int32), rr[:, 2:6], cams, 250)

    def cayley(seg):                                   # optimization.cc:34-70
        l = (seg[3:] - seg[:3]) / np.linalg.norm(seg[3:] - seg[:3])
        m = np.cross(0.5 * (seg[:3] + seg[3:]), l)
        Q = np.stack([l, m / np.linalg.norm(m), np.cross(l, m) / np.linalg.norm(np.cross(l, m))], 1)
        S = (Q - np.eye(3)) @ np.linalg.inv(Q + np.eye(3))
        return np.array([np.linalg.norm(m), S[2, 1], S[0, 2], S[1, 0]])
    tot0 = tot1 = tot2 = 0.0
    for k in range(len(sel)):
        rc, xy = rr[p2[k]:p2[k + 1], 0].astype(int), rr[p2[k]:p2[k + 1], 2:6]
        x0, x1 = cayley(b[k]), cayley(out[k])
        c0, c1 = _np_cost(x0, cams, rc, xy), _np_cost(x1, cams, rc, xy)
        c2 = minimize(_np_cost, x1, args=(cams, rc, xy), method="Nelder-Mead", options=dict(xatol=1e-10, fatol=1e-12, maxiter=2000)).fun
        tot0 += c0; tot1 += c1; tot2 += c2
    assert abs(tot0 - summ[1]) < 1e-6 * tot0 and abs(tot1 - summ[2]) < 1e-6 * tot1        # same cost function, independently coded
    # Ceres stops on the relative change of the TOTAL cost (function_tolerance 1e-6), so single lines keep a little slack
    assert tot1 < 0.85 * tot0 and tot1 - tot2 < 1e-3 * tot1


def test_oracle_optimizer_edge_cases(oracle):
    fn = oracle.lib().orc_optimize_lines
    cams = np.zeros((1, 16)); cams[0, [0, 4, 8]] = 1; cams[0, 12:16] = (1000, 1000, 500, 400)
    seg = np.array([[0.3, 0.2, 5.0, 0.8, 0.25, 5.5]])
    # a line without residuals, and max_iter = 0, stay where they are (unit direction around the old mid point)
    for ptr, it in (([0, 0], 250), ([0, 1], 0)):
        out, valid, summ = oracle.optimize_lines(fn, seg, ptr, [0] * ptr[1], np.array([[100., 100, 300, 120]] * ptr[1]).reshape(-1, 4), cams, it)
        mid = 0.5 * (seg[0, :3] + seg[0, 3:])
        assert valid[0] == 1 and np.allclose(0.5 * (out[0, :3] + out[0, 3:]), mid, atol=1e-9) and abs(np.linalg.norm(out[0, :3] - out[0, 3:]) - 2) < 1e-9
        d = (seg[0, 3:] - seg[0, :3]) / np.linalg.norm(seg[0, 3:] - seg[0, :3])
        assert abs(abs(((out[0, :3] - out[0, 3:]) / 2) @ d) - 1) < 1e-9
    out, valid, summ = oracle.optimize_lines(fn, np.zeros((0, 6)), [0], [], np.zeros((0, 4)), cams, 10)
    assert len(out) == 0


@pytest.mark.parametrize("use_gpu", [1, 0])
def test_oracle_pipeline_with_bundling(oracle, use_gpu):
    sc = synth.make_scene(10, 250, 9, "ring3", noise_px=1.0)
    d = {}
    for uc in (False, True):
        P = oracle.OraclePipeline(False, use_gpu)
        P.add_scene(sc); P.match_images()
        assert P.reconstruct(3, False, -1.0, uc) == 0
        s = P.segments3d()
        d[uc] = (P.num_lines(), np.mean(np.concatenate([_dist_to_gt(s["p1"], sc.lines3d), _dist_to_gt(s["p2"], sc.lines3d)])))
        if uc:
            sm = P.opt_summary()
            assert sm[3] == 0 and sm[2] < sm[1] and sm[5] > 100
    assert abs(d[True][0] - d[False][0]) <= 2 and d[True][1] < d[False][1]          # closer to the ground-truth lines


# ---------------------------------------------------------------------------------------------- cluster -> 3D segments (SURVEY §8f-1)
def test_oracle_cluster_tail_reproduces_the_reference_result_file(oracle):
    """findCollinearSegments(cluster) + project2DsegmentOnto3Dline (line3D.cc:2221-2266, 2342-2452) on the reference's OWN
    clusters: from the line and the 2D residuals listed in testdata/Line3D++_ref/*.txt the oracle rebuilds every one of the
    2501 3D segments of that file (end points to the text rounding); the few extra segments are the tiny ones the
    reference removes afterwards (filterTinySegments needs the cluster's reference view, which the file does not record)."""
    from tests import nvm_util as nu
    inp = nu.load_inputs()
    cam_segs, clusters = nu.fixture_clusters()
    P = oracle.OraclePipeline(True, 1)
    for i in range(inp["V"]):
        w, h = inp["wh"][i]
        assert P.add_view(i, int(w), int(h), inp["K"][i], inp["R"][i], inp["t"][i], inp["median_depth"][i], inp["wps"][i], cam_segs[i]) == 0
    out = np.zeros((64, 6))
    L = oracle.lib()

    def run(cl):
        n = L.orc_collinear_from_cluster(P.ctx, oracle._p(np.ascontiguousarray(cl["p1p2"])), len(cl["cams"]), oracle._p(cl["cams"]), oracle._p(cl["segs"]),
                                         oracle._p(out), 64)
        return out[:n].copy()
    total, matched, extra, worst = nu.check_fixture_segments(run, clusters)
    assert total == 2501 and matched == total and worst < 5e-5, (total, matched, worst)
    assert extra <= 0.02 * total, extra


def test_cpp_frontend_compiles_against_the_public_headers(tmp_path):
    """the drop-in boundary is plain C++: examples/vsfm_frontend.cpp (the reference's main_vsfm.cpp flow on include/line3d.h +
    include/line3d_io.h) must compile warning-free with g++ alone, link against the in-tree library and - without a GPU - fail
    loudly instead of computing on the CPU"""
    from line3dpp_b200 import build
    so = build.build()
    exe = tmp_path / "vsfm_frontend"
    cmd = ["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", os.path.join(ROOT, "examples", "vsfm_frontend.cpp"), "-I" + os.path.join(ROOT, "include"),
           "-L" + os.path.dirname(so), "-ll3d_b200", "-Wl,-rpath," + os.path.dirname(so), "-o", str(exe)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    nvm = tmp_path / "m.nvm"
    nvm.write_text("NVM_V3\n\n1\nimg0.jpg 1000 1 0 0 0 0 0 0 0 0\n\n1\n0 0 5 255 255 255 1 0 0 1.0 2.0\n")
    r = subprocess.run([str(exe), str(nvm), str(tmp_path), str(tmp_path)], capture_output=True, text=True)
    import torch
    if torch.cuda.is_available():
        assert r.returncode == 1 and "fewer than three usable images" in r.stderr, (r.returncode, r.stderr)
    else:
        assert r.returncode == 3 and "no usable CUDA device" in r.stderr, (r.returncode, r.stderr)



def test_reference_addimage_signature_compiles_against_eigen_opencv_headers(tmp_path):
    """include/line3d.h offers the reference's own addImage signature (line3D.h:104-108) when Eigen and OpenCV headers are on the
    include path.  Neither is installed here: compile against the stand-ins of oracle/ref_shim (the headers the verbatim reference
    build uses), link against the in-tree library and check that a view without segments is rejected, not detected on the CPU."""
    from line3dpp_b200 import build
    so = build.build()
    src = tmp_path / "facade.cpp"
    src.write_text(r"""
#include "line3d.h"
#ifndef L3DPP_WITH_EIGEN_OPENCV
#error "the Eigen / OpenCV overloads were not enabled"
#endif
#include <cstdio>
int main() {
    try {
        L3DPP::Line3D L("/tmp", true, -1, 3000, false, true);
        cv::Mat img(2304, 3072, CV_8U);
        Eigen::Matrix3d K = Eigen::Matrix3d::Identity(), R = Eigen::Matrix3d::Identity();
        Eigen::Vector3d t(0, 0, 1);
        std::list<unsigned int> nb; nb.push_back(1);
        std::vector<cv::Vec4f> segs(1, cv::Vec4f(1.f, 2.f, 300.f, 400.f));
        bool a = L.addImage(0u, img, K, R, t, 4.0f, nb, segs);
        bool b = L.addImage(1u, img, K, R, t, 4.0f, nb);          // no segments: rejected (no LSD here)
        std::printf("%d %d %zu\n", int(a), int(b), L.numImages());
        return (a && !b && L.numImages() == 1) ? 0 : 1;
    } catch (const std::exception& e) { std::printf("no GPU: %s\n", e.what()); return 3; }
}
""")
    exe = tmp_path / "facade"
    shim = os.path.join(ROOT, "oracle", "ref_shim")
    cmd = ["g++", "-std=c++17", "-Wall", "-Werror", str(src), "-I" + os.path.join(ROOT, "include"), "-I" + shim, "-L" + os.path.dirname(so), "-ll3d_b200",
           "-Wl,-rpath," + os.path.dirname(so), "-o", str(exe)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    import torch
    assert r.returncode == (0 if torch.cuda.is_available() else 3), (r.returncode, r.stdout, r.stderr)


def test_no_cpu_fallback_without_gpu():
    """without a CUDA device the product must fail loudly, not compute on the CPU"""
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from line3dpp_b200 import capi, line3d
    h = ctypes.c_void_p()
    assert capi.lib().l3d_ctx_create(0, ctypes.byref(h)) < 0 and not h
    with pytest.raises(capi.L3DError):
        capi.Context(0)
    with pytest.raises(capi.L3DError):
        line3d.Line3D(False, True)


def test_product_never_imports_the_oracle():
    for root, _, files in os.walk(os.path.join(ROOT, "line3dpp_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cc", ".h")):
                for line in open(os.path.join(root, f)):
                    if re.match(r"\s*(#\s*include|import|from)\b", line) or "CDLL" in line or "dlopen" in line:
                        assert "oracle" not in line, (f, line)


# ---------------------------------------------------------------------------------------------- BASELINE configs[0]: vsfm_result.nvm on the CPU path
def test_nvm_cpu_reference_run_matches_fixture_statistically(oracle):
    """testdata/vsfm_result.nvm, 26 views, default parameters (README.md:214-221), segments from cv2's LSD (committed
    inputs, tests/golden/make_nvm_inputs.py).  The oracle's restatement of the reference pipeline must reproduce the
    reference's own result testdata/Line3D++_ref statistically: line count within 3 %, symmetric chamfer distance of
    points sampled on the 3D segments below 0.5 % of the scene depth (median) - the same order as the distance between
    the oracle's REF_GPU and REF_CPU semantics.  Index parity is impossible here (different LSD build, SURVEY.md §4)."""
    from tests import nvm_util as nu
    oracle.set_threads(os.cpu_count() or 1)
    inp = nu.load_inputs()
    fx, fl, fr = nu.load_fixture()
    P = oracle.OraclePipeline(True, 1)
    nu.add_all(P.add_view, inp)
    assert P.match_images() == 0 and P.reconstruct(3, False) == 0
    oracle.set_threads(1)
    n_ref = len(set(fl.tolist()))
    assert abs(P.num_lines() - n_ref) <= 0.03 * n_ref, (P.num_lines(), n_ref)
    assert abs(len(P.residuals()) - len(fr)) <= 0.05 * len(fr)
    s = P.segments3d()
    mine = np.concatenate([s["p1"], s["p2"]], 1)
    a, b = nu.sample_points(mine), nu.sample_points(fx)
    depth = float(np.median(inp["median_depth"]))
    m1, p1 = nu.chamfer(a, b)
    m2, p2 = nu.chamfer(b, a)
    assert m1 < 0.005 * depth and m2 < 0.005 * depth, (m1, m2)
    assert p1 < 0.02 * depth and p2 < 0.02 * depth, (p1, p2)


def test_bench_helpers_without_gpu():
    """bench.py's bookkeeping helpers (HBM peak, nominal FP32 peak) never raise: without a GPU they yield None"""
    import importlib.util
    spec = importlib.util.spec_from_file_location("bench_mod", os.path.join(ROOT, "bench.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    assert b.load_peaks()["hbm_gbs"] > 0
    assert b.nominal_fp32_tflops(None) is None
    v = b.nominal_fp32_tflops({"sm_mhz": 1965.0})        # None without a CUDA device, SMs x 128 x 2 x clock with one
    assert v is None or 50.0 < v < 100.0
