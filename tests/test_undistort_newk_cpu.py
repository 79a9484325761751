"""Undistortion into a new camera matrix and size without a GPU: the host restatements of cv2.getOptimalNewCameraMatrix and
cv2.fisheye.estimateNewCameraMatrixForUndistortRectify (csrc/line3d_newk.cc) against the matrices and ROIs OpenCV computed
(tests/golden/ref_undistort_newk_v1.npz), and the map restatement (tests/newk_model.py) against cv2's maps and remaps (DESIGN.md §4a)."""
import os

import numpy as np
import pytest

from line3dpp_b200 import line3d
from tests import lens_model as lm
from tests import newk_model as nm
from tests import undistort_model as um

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_undistort_newk_v1.npz")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLDEN)


def _cases(model=None):
    g = np.load(GOLDEN)
    return [str(n) for n in g["cases"] if model is None or int(g[f"{n}/model"]) == model]


def _host_new_k(g, name):
    """(newK, roi or None) from the host functions, with the arguments cv2 was given"""
    w, h, c, K, model, k, p, _, _ = nm.case_params(g, name)
    lens = nm.lens_dict(model, k, p)
    ns = tuple(int(v) for v in g[f"{name}/new_size_arg"])
    if model == lm.FISHEYE:
        return line3d.fisheye_new_camera_matrix(K, lens, (w, h), float(g[f"{name}/balance"]), ns, float(g[f"{name}/fov_scale"])), None
    return line3d.optimal_new_camera_matrix(K, lens, (w, h), float(g[f"{name}/alpha"]), ns, bool(g[f"{name}/center"]))


@pytest.mark.parametrize("name", _cases())
def test_host_new_camera_matrix_is_opencvs(gold, name):
    newK, roi = _host_new_k(gold, name)
    cv = gold[f"{name}/cv_newK"]
    assert np.abs(newK - cv).max() <= 1e-9 * np.abs(cv).max(), (newK, cv)
    if roi is not None:
        assert roi == tuple(int(v) for v in gold[f"{name}/cv_roi"])


@pytest.mark.parametrize("name", _cases())
def test_model_plus_corrections_is_opencvs_map(gold, name):
    w, h, c, K, model, k, p, newK, (ow, oh) = nm.case_params(gold, name)
    xy, fr = nm.newk_maps(ow, oh, K, newK, model, k, p)
    assert xy.shape == (oh, ow, 2)
    cxy, cfr = um.apply_corrections(xy, fr, gold[f"{name}/diff_idx"], gold[f"{name}/diff_xy"], gold[f"{name}/diff_frac"])
    assert um.sha(cxy, cfr) == str(gold[f"{name}/cv_map_sha"])


@pytest.mark.parametrize("name", _cases())
def test_every_correction_is_one_step(gold, name):
    w, h, c, K, model, k, p, newK, (ow, oh) = nm.case_params(gold, name)
    xy, fr = nm.newk_maps(ow, oh, K, newK, model, k, p)
    idx = gold[f"{name}/diff_idx"]
    fx = lambda a, f: a.astype(np.int64) * 32 + (f & 31).astype(np.int64)
    fy = lambda a, f: a.astype(np.int64) * 32 + (f >> 5).astype(np.int64)
    a, b = xy.reshape(-1, 2)[idx], fr.reshape(-1)[idx]
    ca, cb = gold[f"{name}/diff_xy"], gold[f"{name}/diff_frac"]
    assert (np.abs(fx(a[:, 0], b) - fx(ca[:, 0], cb)) <= 1).all() and (np.abs(fy(a[:, 1], b) - fy(ca[:, 1], cb)) <= 1).all()


def test_differing_entry_counts():
    """what DESIGN.md §4a states: on every case the restatement, cofactor inverse and all, is cv2's map entry for entry (cv::fisheye
    inverts newK by SVD; on these cases that costs nothing)"""
    g = np.load(GOLDEN)
    assert {n: len(g[f"{n}/diff_idx"]) for n in _cases()} == {n: 0 for n in _cases()}


@pytest.mark.parametrize("name", _cases())
def test_restated_remap_reproduces_cv2(gold, name):
    w, h, c, K, model, k, p, newK, (ow, oh) = nm.case_params(gold, name)
    if ow * oh > 2_000_000:
        pytest.skip("the full-size cases are covered on the GPU; the restated remap is checked on the smaller ones")
    img = um.make_image(h, w, c, seed=200 + _cases().index(name))
    xy, fr = nm.newk_maps(ow, oh, K, newK, model, k, p)
    assert um.sha(um.remap(img, xy, fr)) == str(gold[f"{name}/model_remap_sha"])
    cxy, cfr = um.apply_corrections(xy, fr, gold[f"{name}/diff_idx"], gold[f"{name}/diff_xy"], gold[f"{name}/diff_frac"])
    assert um.sha(um.remap(img, cxy, cfr)) == str(gold[f"{name}/cv_remap_sha"])


def test_new_k_equal_to_k_is_the_lens_model(gold):
    """newK = K at the source size is tests/lens_model.py's map, bit for bit, for both models"""
    for name in ("rational8_a0", "fisheye_fov"):
        w, h, c, K, model, k, p, _, _ = nm.case_params(gold, name)
        a = nm.newk_maps(w, h, K, K, model, k, p)
        b = lm.lens_maps(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2], model, k, p)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), name


def test_int16_case_wraps_under_the_new_k(gold):
    """the fisheye case whose source coordinates pass int16 under its new K: cv2's map is the wrapped one, not the saturated one"""
    w, h, c, K, model, k, p, newK, (ow, oh) = nm.case_params(gold, "fisheye_int16")
    assert not np.allclose(newK, K)
    iu, iv = nm.fisheye_uv(ow, oh, K, newK, k)
    wrapped, saturated = lm.maps_wrapped(iu, iv), um.maps_from_uv(iu, iv)
    assert (iu >> 5).max() > 32767 and not np.array_equal(wrapped[0], saturated[0])
    assert um.sha(*wrapped) == str(gold["fisheye_int16/cv_map_sha"])


def test_cases_cover_what_the_contract_names(gold):
    names = _cases()
    radtan, fisheye = _cases(lm.RADTAN), _cases(lm.FISHEYE)
    assert {float(gold[f"{n}/alpha"]) for n in radtan} == {0.0, 0.5, 1.0}
    assert {float(gold[f"{n}/balance"]) for n in fisheye} == {0.0, 0.5, 1.0}
    assert any(float(gold[f"{n}/fov_scale"]) != 1.0 for n in fisheye) and any(bool(gold[f"{n}/center"]) for n in radtan)
    assert {bool(gold[f"{n}/k"][3:].any()) for n in radtan} == {False, True}
    out = [(tuple(gold[f"{n}/size"][:2]), tuple(gold[f"{n}/out_size"])) for n in names]
    assert any(o[0] < s[0] for s, o in out) and any(o[0] > s[0] for s, o in out)
    assert any(o[0] * s[1] != o[1] * s[0] for s, o in out)
    assert {int(gold[f"{n}/size"][2]) for n in names} == {1, 3}


def test_host_functions_against_live_cv2():
    """a sweep beyond the golden cases, where cv2 is installed: other lenses, alphas, balances, sizes and off-centre cameras"""
    cv2 = pytest.importorskip("cv2")
    K = np.array([[2500.0, 0, 1536.3], [0, 2480.0, 1151.7], [0, 0, 1]])
    for k, p in (((-0.2, 0.05, 0.01, 0, 0, 0), (0.001, -0.0007)), ((0.12, -0.05, 0.01, 0.08, -0.02, 0.005), (0.0007, -0.0004)),
                 ((-0.2, 0, 0, 0, 0, 0), (0, 0))):
        dist = np.array([k[0], k[1], p[0], p[1], k[2], k[3], k[4], k[5]])
        for alpha in (0.0, 0.25, 1.0):
            for ns in ((0, 0), (2000, 1500), (4000, 2000)):
                for center in (False, True):
                    M, roi = cv2.getOptimalNewCameraMatrix(K, dist, (3072, 2304), alpha, ns, centerPrincipalPoint=center)
                    M2, roi2 = line3d.optimal_new_camera_matrix(K, nm.lens_dict(0, k, p), (3072, 2304), alpha, ns, center)
                    assert np.abs(M2 - M).max() <= 1e-9 * np.abs(M).max() and roi2 == tuple(roi), (k, alpha, ns, center)
    for Kf in (np.array([[800.0, 0, 1536], [0, 800, 1152], [0, 0, 1]]), np.array([[805.3, 0, 1530.7], [0, 790.2, 1160.1], [0, 0, 1]])):
        D = np.array([0.05, -0.01, 0.002, -0.0005])
        for b in (0.0, 0.3, 1.0, 1.5):
            for ns in ((0, 0), (2000, 1500), (4000, 2000)):
                for fs in (1.0, 1.3, 0.7):
                    P = cv2.fisheye.estimateNewCameraMatrixForUndistortRectify(Kf, D, (3072, 2304), np.eye(3), balance=b, new_size=ns, fov_scale=fs)
                    P2 = line3d.fisheye_new_camera_matrix(Kf, nm.lens_dict(1, list(D) + [0, 0], (0, 0)), (3072, 2304), b, ns, fs)
                    assert np.abs(P2 - P).max() <= 1e-9 * np.abs(P).max(), (b, ns, fs)


def test_fold_cases_bound_the_outer_box_by_the_border():
    """the folding-lens cases pin getOptimalNewCameraMatrix's outer rectangle: some interior grid point undistorts outside the bounding
    box of the 32 border points, so a box over all 81 points would give another matrix"""
    cv2 = pytest.importorskip("cv2")
    g = np.load(GOLDEN)
    for name in ("rational8_fold_a05", "rational8_fold_a1_center"):
        w, h, c, K, model, k, p, _, _ = nm.case_params(g, name)
        grid = np.array([(x * (w - 1) / 8, y * (h - 1) / 8) for y in range(9) for x in range(9)], np.float64)
        dist = np.array([k[0], k[1], p[0], p[1], k[2], k[3], k[4], k[5]])
        q = cv2.undistortPoints(grid.reshape(-1, 1, 2), K, dist).reshape(9, 9, 2)
        border = np.concatenate([q[0], q[8], q[:, 0], q[:, 8]])
        assert (q.reshape(-1, 2).min(0) < border.min(0)).any() or (q.reshape(-1, 2).max(0) > border.max(0)).any(), name


def test_optimal_new_camera_matrix_on_random_cameras_against_live_cv2():
    """240 seeded random radtan cameras (5 and 8 coefficients, off-centre principal points, alphas, sizes, centerPrincipalPoint),
    strong enough that some lenses fold over: every matrix within 1e-9 relative of cv2's and every ROI equal"""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(11)
    for t in range(240):
        w, h = int(rng.integers(300, 3000)), int(rng.integers(300, 3000))
        f = rng.uniform(0.4, 1.5) * max(w, h)
        K = np.array([[f, 0, w / 2 + rng.uniform(-0.1, 0.1) * w], [0, f * rng.uniform(0.9, 1.1), h / 2 + rng.uniform(-0.1, 0.1) * h], [0, 0, 1]])
        k = list(rng.uniform(-0.5, 0.5, 3)) + (list(rng.uniform(-0.5, 0.5, 3)) if rng.random() < 0.5 else [0.0, 0.0, 0.0])
        p = list(rng.uniform(-0.01, 0.01, 2))
        dist = np.array([k[0], k[1], p[0], p[1], k[2], k[3], k[4], k[5]])
        alpha = float(rng.choice([0.0, 0.3, 0.5, 1.0]))
        ns = [(0, 0), (int(w * 0.7), int(h * 0.9))][int(rng.integers(2))]
        center = bool(rng.integers(2))
        M, roi = cv2.getOptimalNewCameraMatrix(K, dist, (w, h), alpha, ns, centerPrincipalPoint=center)
        M2, roi2 = line3d.optimal_new_camera_matrix(K, nm.lens_dict(0, k, p), (w, h), alpha, ns, center)
        assert np.abs(M2 - M).max() <= 1e-9 * np.abs(M).max() and roi2 == tuple(int(v) for v in roi), (t, M, M2, roi, roi2)


def test_new_k_and_out_size_take_one_value_or_one_per_image():
    """Context.undistort's new_K and out_size, like K: one value for all images (a list, tuple or array) or one entry per image"""
    from line3dpp_b200.capi import _one_or_per_image as f
    K = [[1.0, 0, 2], [0, 1, 3], [0, 0, 1]]
    assert f(K, 3, 2) == [K] * 3 and len(f(np.eye(3), 2, 2)) == 2 and f(None, 2, 2) == [None, None]
    per = f([None, np.eye(3)], 2, 2)
    assert per[0] is None and per[1].shape == (3, 3)
    assert f([10, 20], 2, 1) == [[10, 20]] * 2 and f((10, 20), 3, 1) == [(10, 20)] * 3 and f(np.array([10, 20]), 2, 1)[1].tolist() == [10, 20]
    assert f([None, None], 2, 1) == [None, None] and f([(1, 2), None], 2, 1) == [(1, 2), None] and f([(1, 2), (3, 4)], 2, 1) == [(1, 2), (3, 4)]


def test_host_functions_reject_the_other_lens_and_bad_cameras():
    K = np.array([[500.0, 0, 320], [0, 500, 240], [0, 0, 1]])
    radtan, fisheye = nm.lens_dict(0, [0.1, 0, 0, 0, 0, 0], [0, 0]), nm.lens_dict(1, [0.1, 0, 0, 0, 0, 0], [0, 0])
    with pytest.raises(ValueError):
        line3d.optimal_new_camera_matrix(K, fisheye, (640, 480), 0.0)
    with pytest.raises(ValueError):
        line3d.fisheye_new_camera_matrix(K, radtan, (640, 480))
    for bad_K, size in ((np.diag([0.0, 500, 1]), (640, 480)), (np.diag([np.nan, 500, 1]), (640, 480)), (K, (0, 480)), (K, (640, -1))):
        with pytest.raises(ValueError):
            line3d.optimal_new_camera_matrix(bad_K, radtan, size, 0.0)
        with pytest.raises(ValueError):
            line3d.fisheye_new_camera_matrix(bad_K, fisheye, size)
    with pytest.raises(ValueError):
        line3d.optimal_new_camera_matrix(K, radtan, (640, 480), 0.0, (-5, 10))
