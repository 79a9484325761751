"""GPU parity of the full hot path (match -> orientation -> score -> inverse -> filter -> affinity -> diffusion ->
clusters -> 3D lines) through the L3DPP::Line3D mirror, against the oracle pipeline.

The oracle's host logic (oracle/l3d_oracle.cc) is driven twice:
  * with the UNMODIFIED reference kernels (-fmad=false) as its accelerator backend -> this IS the reference GPU path
    except for line3D.cc's host glue; the product must agree index-exactly and bit-exactly on overlaps / depths / scores
    (what that run produced on the synthetic scenes: tests/golden/ref_gpu_pipelines_v1.npz, tests/golden/make_ref_gpu_golden.py);
  * with its CPU emulation, to show the same at libm tolerance.
"""
import numpy as np
import pytest

from line3dpp_b200 import capi, synth, line3d
from tests import util

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def scene():
    return synth.make_scene(14, 500, 31, "ring3")


@pytest.fixture(scope="module")
def product(scene):
    L = line3d.Line3D(neighbors_by_worldpoints=False, use_gpu=True)
    L.add_scene(scene)
    L.match_images()
    yield L
    L.close()


@pytest.fixture(scope="module")
def ref_pipe():
    return np.load(util.REF_GPU_PIPELINES)


@pytest.fixture(scope="module")
def oracle_cpu(scene, oracle):
    P = oracle.OraclePipeline(False, True)
    P.add_scene(scene)
    assert P.match_images() == 0
    return P


def _same_matches(a, b, exact_scores):
    assert len(a) == len(b)
    for f in ("src_cam", "src_seg", "tgt_cam", "tgt_seg"):
        assert np.array_equal(a[f], b[f]), f
    for f in ("overlap", "d_p1", "d_p2", "d_q1", "d_q2"):
        assert np.array_equal(util.bits(a[f]), util.bits(b[f])), f
    if exact_scores:
        assert np.array_equal(util.bits(a["score3D"]), util.bits(b["score3D"]))
    else:
        np.testing.assert_allclose(a["score3D"], b["score3D"], rtol=2e-5, atol=2e-6)


def test_view_pairs_and_regularisers(product, ref_pipe, scene):
    assert np.array_equal(product.pairs(), ref_pipe["pipe_pairs"])
    for cam in scene.cam_ids:
        k1, md1 = product.view_info(cam)
        k2, md2 = ref_pipe[f"pipe_vi_{cam}"]
        assert np.float32(k1) == k2 and np.float32(md1) == md2, cam


def test_scored_matches_bit_exact_vs_reference_kernels(product, ref_pipe, scene):
    """all matches of every view right after scoring: order, ids, overlap, depths AND score3D bit-identical"""
    total = 0
    for cam in scene.cam_ids:
        mine = product.view_matches(cam, kept_only=False)
        assert np.array_equal(util.match_sha(mine), ref_pipe[f"pipe_scored_{cam}"]), cam
        total += len(mine)
    assert total > 20000


def test_kept_matches_and_estimates_vs_reference_kernels(product, ref_pipe, scene):
    for cam in scene.cam_ids:
        assert np.array_equal(util.match_sha(product.view_matches(cam, kept_only=True)), ref_pipe[f"pipe_kept_{cam}"]), cam
    best, p = product.estimates()
    assert len(best) == ref_pipe["pipe_est_n"][0] and np.array_equal(util.match_sha(best), ref_pipe["pipe_est_best"])
    np.testing.assert_allclose(p, ref_pipe["pipe_est_p"], rtol=0, atol=1e-12)
    assert len(best) > 2000


def test_scored_matches_vs_cpu_oracle(product, oracle_cpu, scene):
    """same against the pure-CPU emulation: ids/overlap exact, depths/scores at libm tolerance (rsqrt/expf/acosf)"""
    nbad, noff, ntot = 0, 0, 0
    for cam in scene.cam_ids:
        mine = product.view_matches(cam, kept_only=False)
        ref = oracle_cpu.scored(cam)
        if len(mine) != len(ref) or not np.array_equal(mine["tgt_seg"], ref["tgt_seg"]):
            nbad += 1      # a depth sign / orientation / score>0 decision flipped by a 1-ulp libm difference: tolerated, counted
            continue
        assert np.array_equal(util.bits(mine["overlap"]), util.bits(ref["overlap"]))
        np.testing.assert_allclose(mine["d_p1"], ref["d_p1"], rtol=1e-3)
        # a similarity that sits at the 0.5 truncation (cudawrapper.cu:346) can flip with a 1-ulp expf difference and
        # moves the scores of that segment's matches by up to 0.5: allow a small fraction of outliers
        off = ~np.isclose(mine["score3D"], ref["score3D"], rtol=1e-3, atol=1e-4)
        noff += int(off.sum()); ntot += len(off)
        assert np.abs(mine["score3D"] - ref["score3D"])[off].max(initial=0) <= 1.0
    assert nbad <= 3 and ntot > 10000 and noff / ntot < 0.01


@pytest.mark.parametrize("diffusion", [False, True])
def test_reconstruction_vs_reference_kernels(scene, ref_pipe, diffusion):
    """affinity matrix before diffusion and the one handed to the clustering: same local ids, same edges in the same order,
    weights to libm tolerance; 3D lines: same residuals, end points within 1e-6 scene units (stated tolerance)"""
    L = line3d.Line3D(neighbors_by_worldpoints=False, use_gpu=True)
    L.add_scene(scene)
    L.match_images()
    L.reconstruct_3d_lines(3, diffusion)
    st = L.stats()
    assert st["lines3D"] > 100
    util.check_reconstruction(ref_pipe, f"rec_{int(diffusion)}_", L.local2global(), L.affinity(raw=True), L.affinity(raw=False), st["lines3D"],
                              L.residuals(), L.segments3d(), 1e-6)
    L.close()


def rdd_graph():
    """a random symmetric affinity graph as the CLEdge list A_: (n, ei, ej, ew)"""
    rng = np.random.default_rng(3)
    n = 3000
    a = rng.integers(0, n, 40000); b = rng.integers(0, n, 40000)
    keep = a != b
    a, b = a[keep], b[keep]
    key = np.minimum(a, b) * n + np.maximum(a, b)
    _, idx = np.unique(key, return_index=True)
    a, b = a[np.sort(idx)], b[np.sort(idx)]
    # every node needs at least one edge (the reference kernel reads start index -1 otherwise)
    missing = np.setdiff1d(np.arange(n), np.concatenate([a, b]))
    a = np.concatenate([a, missing]); b = np.concatenate([b, (missing + 1) % n])
    w = rng.uniform(0.5, 1.0, len(a)).astype(np.float32)
    ei = np.stack([a, b], 1).reshape(-1).astype(np.int32)       # (i,j),(j,i) consecutive like A_
    ej = np.stack([b, a], 1).reshape(-1).astype(np.int32)
    ew = np.repeat(w, 2)
    return n, ei, ej, ew


def test_rdd_bit_exact_vs_reference(gpu_ctx, oracle):
    """l3d_rdd == verbatim SparseMatrix + replicator_dynamics_diffusion_GPU on a random symmetric affinity graph (its result:
    tests/golden/ref_gpu_kernels_v1.npz, tests/golden/make_ref_gpu_golden.py)"""
    import ctypes as C
    n, ei, ej, ew = rdd_graph()
    gold = np.load(util.REF_GPU_GOLDEN)
    L = gpu_ctx.L
    oi, oj, ow = np.zeros_like(ei), np.zeros_like(ej), np.zeros_like(ew)
    ms = C.c_float(0)
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    rc = L.l3d_rdd(gpu_ctx.h, n, C.c_longlong(len(ei)), p(ei), p(ej), p(ew), 10, p(oi), p(oj), p(ow), C.byref(ms))
    assert rc == 0
    assert np.array_equal(util.sha(oi, oj, util.bits(ow)), gold["rdd_sha"])
    ci, cj, cw, _ = oracle.rdd(oracle.lib().orc_rdd_f32, ei, ej, ew, n)
    assert np.array_equal(util.sha(ci, cj, util.bits(cw)), gold["rdd_sha"])     # pins the CPU restatement too


# ---------------------------------------------------------------------------------------------- BASELINE configs[1]: vsfm_result.nvm on 1 GPU
def test_nvm_b200_vs_reference_kernels_and_fixture():
    """testdata/vsfm_result.nvm through L3DPP::Line3D on the GPU (neighbours from world points, default parameters):
    index-exact against the oracle host logic driving the UNMODIFIED reference kernels (its results: tests/golden/ref_gpu_nvm_v1.npz),
    3D endpoints within 1e-6 scene units, and statistically equal to the reference's own result fixture testdata/Line3D++_ref."""
    from tests import nvm_util as nu
    inp = nu.load_inputs()
    fx, fl, fr = nu.load_fixture()
    L = line3d.Line3D(neighbors_by_worldpoints=True, use_gpu=True)
    nu.add_all(L.add_image, inp)
    L.match_images()
    L.reconstruct_3d_lines(3, False)
    g = np.load(util.REF_GPU_NVM)
    assert np.array_equal(L.pairs(), g["nvm_pairs"])
    for cam in range(inp["V"]):
        assert np.array_equal(util.match_sha(L.view_matches(cam, kept_only=True)), g[f"nvm_kept_{cam}"]), cam
    assert np.array_equal(util.sha(np.asarray(L.local2global(), np.int64).reshape(-1)), g["nvm_l2g"])
    st = L.stats()
    assert st["lines3D"] == g["nvm_lines"][0]
    mr = L.residuals()
    assert np.array_equal(util.sha(np.asarray(mr["cam"], np.int64), np.asarray(mr["seg"], np.int64)), g["nvm_res_cam_seg"])
    ms = L.segments3d()
    a = np.sort(np.stack([ms["p1"], ms["p2"]], 1), axis=1)
    np.testing.assert_allclose(a, g["nvm_seg_pts"], atol=1e-6)
    # statistical comparison with the reference's own output
    n_ref = len(set(fl.tolist()))
    assert abs(st["lines3D"] - n_ref) <= 0.03 * n_ref, (st["lines3D"], n_ref)
    mine = np.concatenate([ms["p1"], ms["p2"]], 1)
    depth = float(np.median(inp["median_depth"]))
    m1, _ = nu.chamfer(nu.sample_points(mine), nu.sample_points(fx))
    m2, _ = nu.chamfer(nu.sample_points(fx), nu.sample_points(mine))
    assert m1 < 0.005 * depth and m2 < 0.005 * depth, (m1, m2)
    print("nvm on the GPU:", st)
    import ctypes as C
    buf = C.create_string_buffer(512)
    assert L.L.l3dpp_output_filename(L.h, buf, 512) > 0
    assert buf.value.decode() == "Line3D++__W_FULL__N_10__sigmaP_2.5__sigmaA_10__epiOverlap_0.25__kNN_10__vis_3"      # the reference's own file name
    L.close()


def test_cluster_tail_reproduces_the_reference_result_file():
    """the host-side cluster -> 3D segment tail of the product (csrc/line3d_host.cc, findCollinearSegments line3D.cc:2342-2452)
    rebuilds every 3D segment of the reference's own result file from its lines + residuals"""
    import ctypes as C
    from tests import nvm_util as nu
    inp = nu.load_inputs()
    cam_segs, clusters = nu.fixture_clusters()
    L = line3d.Line3D(neighbors_by_worldpoints=True, use_gpu=True)
    for i in range(inp["V"]):
        w, h = inp["wh"][i]
        L.add_image(i, int(w), int(h), inp["K"][i], inp["R"][i], inp["t"][i], inp["median_depth"][i], inp["wps"][i], cam_segs[i])
    out = np.zeros((64, 6))
    p = lambda a: a.ctypes.data_as(C.c_void_p)

    def run(cl):
        n = L.L.l3dpp_collinear_from_cluster(L.h, p(np.ascontiguousarray(cl["p1p2"])), len(cl["cams"]), p(cl["cams"]), p(cl["segs"]), p(out), 64)
        return out[:n].copy()
    total, matched, extra, worst = nu.check_fixture_segments(run, clusters)
    assert total == 2501 and matched == total and worst < 5e-5, (total, matched, worst)
    assert extra <= 0.02 * total, extra
    L.close()


def test_writers_reproduce_the_reference_result_files_byte_for_byte(tmp_path):
    """save3DLinesAsTXT / saveResultAsOBJ / saveResultAsSTL (line3D.cc:2465-2687) against the reference's own files
    testdata/Line3D++_ref/*.{txt,obj,stl}: the lines parsed from those files are fed back into L3DPP::Line3D and the three
    writers must reproduce them byte for byte (SHA-256 committed by tests/golden/make_writer_golden.py); the file name of the
    nvm configuration is checked in test_nvm_b200_vs_reference_kernels_and_fixture"""
    import ctypes as C
    import hashlib
    import os
    from tests import nvm_util as nu
    inp = nu.load_inputs()
    segs3d, seg_line, res = nu.load_fixture()
    gold = np.load(os.path.join(nu.G, "ref_writers_v1.npz"))
    L = line3d.Line3D(neighbors_by_worldpoints=True, use_gpu=True)
    for i in range(inp["V"]):                           # views whose 2D segments sit at the reference's own segment ids
        r = res[res[:, 1] == i]
        lines = np.zeros((int(r[:, 2].max()) + 1 if len(r) else 1, 4), np.float32)
        lines[r[:, 2].astype(int)] = r[:, 3:7]
        w, h = inp["wh"][i]
        L.add_image(i, int(w), int(h), inp["K"][i], inp["R"][i], inp["t"][i], inp["median_depth"][i], inp["wps"][i], lines)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    ids = sorted(set(seg_line.tolist()))
    nseg = np.array([(seg_line == ln).sum() for ln in ids], np.int32)
    nres = np.array([(res[:, 0] == ln).sum() for ln in ids], np.int32)
    order = np.argsort(res[:, 0], kind="stable")
    rc, rs = np.ascontiguousarray(res[order, 1], np.uint32), np.ascontiguousarray(res[order, 2], np.uint32)

    def written(segs, save, ext):
        assert L.L.l3dpp_set_lines(L.h, len(ids), p(nseg), p(np.ascontiguousarray(segs, np.float64)), p(nres), p(rc), p(rs)) == 0
        d = tmp_path / ext
        d.mkdir()
        assert save(L.h, str(d).encode()) == 0
        files = os.listdir(d)
        assert len(files) == 1 and files[0].endswith("." + ext)
        return hashlib.sha256(open(d / files[0], "rb").read()).hexdigest()
    assert len(gold["stl_segs"]) == len(segs3d) == nseg.sum()
    assert written(segs3d, L.L.l3dpp_save_txt, "txt") == str(gold["sha_txt"])
    assert written(segs3d, L.L.l3dpp_save_obj, "obj") == str(gold["sha_obj"])
    assert written(gold["stl_segs"], L.L.l3dpp_save_stl, "stl") == str(gold["sha_stl"])
    L.close()


def test_add_image_and_writer_errors_are_reported(tmp_path):
    """ADVICE r1: addImage failures are attributable (status + sticky lastError), writers report unwritable folders"""
    sc = synth.make_scene(6, 200, 3, "ring2")
    L = line3d.Line3D(neighbors_by_worldpoints=False, use_gpu=True)
    L.add_scene(sc)
    import ctypes as C
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    K, R, t = np.ascontiguousarray(sc.K[0]), np.ascontiguousarray(sc.R[0]), np.ascontiguousarray(sc.t[0])
    nb, sg = np.ascontiguousarray(sc.neighbors[0], np.uint32), np.ascontiguousarray(sc.segs[0], np.float32)
    add = lambda cam, w: L.L.l3dpp_add_image(L.h, C.c_uint(cam), w, w * 3 // 4, p(K), p(R), p(t), C.c_float(4.0), p(nb), len(nb), p(sg), len(sg))
    assert add(0, 3072) < 0 and b"already in use" in L.L.l3dpp_last_error(L.h)          # duplicate camera id
    assert add(77, 100) < 0 and b"too small" in L.L.l3dpp_last_error(L.h)
    assert add(78, 3072) == 0                                                          # a success ...
    assert b"too small" in L.L.l3dpp_last_error(L.h)                                   # ... does not wipe the earlier failure
    L.match_images()
    L.reconstruct_3d_lines(3, False)
    assert L.stats()["lines3D"] > 20
    with pytest.raises(Exception) as e:
        L.save_txt(str(tmp_path / "does" / "not" / "exist"))
    assert "cannot open" in str(e.value)
    L.save_txt(str(tmp_path))
    assert any(f.name.endswith(".txt") for f in tmp_path.iterdir())
    L.close()


def test_add_image_reports_the_first_failed_check_in_each_overloads_order(tmp_path):
    """a call that fails several checks reports the first: the segments overload checks the size, the neighbours, the segments and
    then the camera ID; the image overload the size, the camera ID and then the neighbours (line3D.cc:116-155)"""
    sc = synth.make_scene(6, 200, 3, "ring2")
    L = line3d.Line3D(neighbors_by_worldpoints=False, use_gpu=True, output_folder=str(tmp_path), load_segments=False)
    L.add_scene(sc)
    K, R, t, nb, sg = sc.K[0], sc.R[0], sc.t[0], sc.neighbors[0], sc.segs[0]

    def error(add):
        with pytest.raises(capi.L3DError) as e:
            add()
        return str(e.value)
    assert "too small" in error(lambda: L.add_image(0, 100, 75, K, R, t, 4.0, [], ()))
    assert "no visual neighbors" in error(lambda: L.add_image(0, 3072, 2304, K, R, t, 4.0, [], sg))
    assert "load_segments is off" in error(lambda: L.add_image(0, 3072, 2304, K, R, t, 4.0, nb, ()))
    assert "no visual neighbors" in error(lambda: L.add_image(77, 3072, 2304, K, R, t, 4.0, [], ()))
    assert "already in use" in error(lambda: L.add_image(0, 3072, 2304, K, R, t, 4.0, nb, sg))
    img = np.zeros((900, 1200), np.uint8)
    assert "too small" in error(lambda: L.add_image_pixels(0, img[:700, :700], K, R, t, 4.0, [], ()))
    assert "already in use" in error(lambda: L.add_image_pixels(0, img, K, R, t, 4.0, [], ()))
    assert "no visual neighbors" in error(lambda: L.add_image_pixels(77, img, K, R, t, 4.0, [], ()))
    with pytest.raises(KeyError):                                                          # nothing was added ...
        L.view_segments(77)
    assert L.view_segments(0).tobytes() == np.ascontiguousarray(sg, np.float32).tobytes()   # ... or replaced
    L.close()
