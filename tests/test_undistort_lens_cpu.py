"""The rational and fisheye restatement (tests/lens_model.py) against what OpenCV computed (tests/golden/ref_undistort_lens_v1.npz):
with the stored corrections it rebuilds cv2's maps exactly, every correction is one 1/32-px step, the restated remap reproduces
cv2.remap, and the rational model with k4 = k5 = k6 = 0 is the pinhole model of tests/undistort_model.py bit for bit."""
import os

import numpy as np
import pytest

from tests import lens_model as lm
from tests import undistort_model as um

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_undistort_lens_v1.npz")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLDEN)


def _cases():
    return [str(n) for n in np.load(GOLDEN)["cases"]]


@pytest.mark.parametrize("name", _cases())
def test_model_plus_corrections_is_opencvs_map(gold, name):
    w, h, c, K, model, k, p = lm.case_params(gold, name)
    xy, fr = lm.model_maps_for(w, h, K, model, k, p)
    cxy, cfr = um.apply_corrections(xy, fr, gold[f"{name}/diff_idx"], gold[f"{name}/diff_xy"], gold[f"{name}/diff_frac"])
    assert um.sha(cxy, cfr) == str(gold[f"{name}/cv_map_sha"])


@pytest.mark.parametrize("name", _cases())
def test_every_correction_is_one_step(gold, name):
    w, h, c, K, model, k, p = lm.case_params(gold, name)
    xy, fr = lm.model_maps_for(w, h, K, model, k, p)
    idx = gold[f"{name}/diff_idx"]
    fx = lambda a, f: a.astype(np.int64) * 32 + (f & 31).astype(np.int64)
    fy = lambda a, f: a.astype(np.int64) * 32 + (f >> 5).astype(np.int64)
    a, b = xy.reshape(-1, 2)[idx], fr.reshape(-1)[idx]
    ca, cb = gold[f"{name}/diff_xy"], gold[f"{name}/diff_frac"]
    assert (np.abs(fx(a[:, 0], b) - fx(ca[:, 0], cb)) <= 1).all() and (np.abs(fy(a[:, 1], b) - fy(ca[:, 1], cb)) <= 1).all()


@pytest.mark.parametrize("name", _cases())
def test_restated_remap_reproduces_cv2(gold, name):
    w, h, c, K, model, k, p = lm.case_params(gold, name)
    if w * h > 2_000_000:
        pytest.skip("the full-size cases are covered on the GPU; the restated remap is checked on the smaller ones")
    img = um.make_image(h, w, c, seed=100 + _cases().index(name))
    xy, fr = lm.model_maps_for(w, h, K, model, k, p)
    assert um.sha(um.remap(img, xy, fr)) == str(gold[f"{name}/model_remap_sha"])
    cxy, cfr = um.apply_corrections(xy, fr, gold[f"{name}/diff_idx"], gold[f"{name}/diff_xy"], gold[f"{name}/diff_frac"])
    assert um.sha(um.remap(img, cxy, cfr)) == str(gold[f"{name}/cv_remap_sha"])


def test_rational_with_zero_k4_k6_is_the_pinhole_model(gold):
    w, h, c, K, model, k, p = lm.case_params(gold, "rational_zero")
    assert model == lm.RADTAN and not k[3:].any()
    a = lm.model_maps_for(w, h, K, model, k, p)
    b = um.undistort_maps(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2], k[0], k[1], k[2], p[0], p[1])
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_int16_case_wraps_where_the_pinhole_path_saturates(gold):
    """the case that decides it: cv::fisheye's (short) cast wraps, and cv2's map agrees with the wrapped model everywhere"""
    w, h, c, K, model, k, p = lm.case_params(gold, "fisheye_int16")
    iu, iv = lm.fisheye_uv(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2], *k[:4])
    wrapped, saturated = lm.maps_wrapped(iu, iv), um.maps_from_uv(iu, iv)
    assert (iu >> 5).max() > 32767 and not np.array_equal(wrapped[0], saturated[0])
    assert um.sha(*wrapped) == str(gold["fisheye_int16/cv_map_sha"])
