"""Lens undistortion without a GPU: the numpy restatement (tests/undistort_model.py) against what OpenCV computed
(tests/golden/ref_undistort_v1.npz, tests/golden/make_undistort_golden.py), and the cv::Mat overload of Line3D::undistortImage
compiled against header stand-ins."""
import os
import subprocess

import numpy as np
import pytest

from tests import undistort_model as um

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_undistort_v1.npz")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLDEN)


def _cases():
    return [str(n) for n in np.load(GOLDEN)["cases"]]


def _opencv_maps(g, name):
    """cv2's maps: the model's with the stored differing entries put in"""
    w, h, c, K, rad, tan = um.case_params(g, name)
    xy, fr = um.model_maps_for(w, h, K, rad, tan)
    return um.apply_corrections(xy, fr, g[f"{name}/diff_idx"], g[f"{name}/diff_xy"], g[f"{name}/diff_frac"])


@pytest.mark.parametrize("name", _cases())
def test_model_map_plus_corrections_is_opencvs_map(gold, name):
    xy, fr = _opencv_maps(gold, name)
    assert um.sha(xy, fr) == str(gold[f"{name}/cv_map_sha"])


@pytest.mark.parametrize("name", _cases())
def test_map_differences_are_single_steps_and_rare(gold, name):
    """OpenCV accumulates x along a row (and by SIMD blocks); the model evaluates the formula per pixel.  Where the two differ, each
    coordinate differs by at most one 1/32-px step, and that happens at no more than 1e-3 of the pixels"""
    w, h, c, K, rad, tan = um.case_params(gold, name)
    iu, iv = um.fixed_point_uv(w, h, float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), *map(float, rad), *map(float, tan))
    idx = gold[f"{name}/diff_idx"]
    assert len(idx) <= 1e-3 * w * h
    if len(idx) == 0:
        return
    cxy, cfr = gold[f"{name}/diff_xy"].astype(np.int64), gold[f"{name}/diff_frac"].astype(np.int64)
    assert (np.abs(cxy) < 32767).all()                    # not saturated: the 1/32-px position can be rebuilt
    du = cxy[:, 0] * 32 + (cfr & 31) - iu.reshape(-1)[idx]
    dv = cxy[:, 1] * 32 + (cfr >> 5) - iv.reshape(-1)[idx]
    assert (np.abs(du) <= 1).all() and (np.abs(dv) <= 1).all() and ((du != 0) | (dv != 0)).all()


@pytest.mark.parametrize("name", _cases())
def test_model_remap_reproduces_opencv(gold, name):
    """the restated remap on cv2's own maps gives cv2.remap's output byte for byte; on the model's maps it gives what cv2.remap
    made of those"""
    w, h, c, K, rad, tan = um.case_params(gold, name)
    img = um.make_image(h, w, c, seed=_cases().index(name))
    assert um.sha(um.remap(img, *_opencv_maps(gold, name))) == str(gold[f"{name}/cv_remap_sha"])
    out = um.remap(img, *um.model_maps_for(w, h, K, rad, tan))
    assert um.sha(out) == str(gold[f"{name}/model_remap_sha"])
    if name == "zero":
        assert np.array_equal(out, img)


def test_model_fix_saturates_like_x86():
    t = np.array([0.5 / 32, 1.5 / 32, -0.5 / 32, 2 ** 26, -2 ** 26 - 1, np.inf, -np.inf, np.nan])
    assert um.fix32(t).tolist() == [0, 2, 0, -2 ** 31, -2 ** 31, -2 ** 31, -2 ** 31, -2 ** 31]


MAT_STANDIN = r"""
// cv::Mat with pixels: the members include/line3d.h's undistortImage overload uses, plus what its addImage overload uses
#pragma once
#include <cstddef>
#include <vector>
#define CV_8UC1 0
#define CV_8UC3 16
namespace cv {
template <class T, int N> struct Vec { T val[N]; T operator()(int i) const { return val[i]; } };
typedef Vec<float, 4> Vec4f;
class Mat {
    std::vector<unsigned char> buf_;
    int type_ = CV_8UC1;
public:
    int rows = 0, cols = 0;
    unsigned char* data = nullptr;
    size_t step = 0;
    int type() const { return type_; }
    int channels() const { return type_ == CV_8UC3 ? 3 : 1; }
    void create(int r, int c, int t) { rows = r; cols = c; type_ = t; step = (size_t)c * channels(); buf_.assign(step * r, 0); data = buf_.data(); }
    void create_padded(int r, int c, int t, size_t s) { create(r, c, t); step = s; buf_.assign(s * r, 0); data = buf_.data(); }
};
}  // namespace cv
"""

FACADE = r"""
#include "line3d.h"
#ifndef L3DPP_WITH_EIGEN_OPENCV
#error "the Eigen / OpenCV overloads were not enabled"
#endif
#include <cstdio>
int main(int, char** argv) {
    const int W = 37, H = 23;
    cv::Mat in, out;
    in.create_padded(H, W, CV_8UC3, 128);                       // row step > cols * channels
    for (int y = 0; y < H; ++y) for (int x = 0; x < W; ++x) for (int c = 0; c < 3; ++c) in.data[y * 128 + 3 * x + c] = (unsigned char)((x * 7 + y * 13 + c * 29) & 255);
    Eigen::Matrix3d K = Eigen::Matrix3d::Identity();
    K(0, 0) = 41.5; K(1, 1) = 40.25; K(0, 2) = 17.75; K(1, 2) = 11.5; K(0, 1) = 0.5;   // the skew is ignored
    try {
        L3DPP::Line3D::undistortImage(in, out, Eigen::Vector3d(-0.21, 0.04, 0.01), Eigen::Vector2d(0.003, -0.002), K);
    } catch (const std::invalid_argument& e) { std::printf("rejected: %s\n", e.what()); return 4; }
    catch (const std::runtime_error& e) { std::printf("no GPU: %s\n", e.what()); return 3; }
    if (out.rows != H || out.cols != W || out.type() != CV_8UC3) return 5;
    FILE* f = std::fopen(argv[1], "wb");
    for (int y = 0; y < H; ++y) std::fwrite(out.data + y * out.step, 1, 3 * W, f);
    std::fclose(f);
    K(0, 0) = 0.0;
    try { L3DPP::Line3D::undistortImage(in, out, Eigen::Vector3d(0, 0, 0), Eigen::Vector2d(0, 0), K); } catch (const std::invalid_argument&) { return 0; }
    return 7;
}
"""


def test_cv_mat_undistort_overload_compiles_and_runs(tmp_path):
    """the reference's signature undistortImage(const cv::Mat&, cv::Mat&, Eigen::Vector3d, Eigen::Vector2d, Eigen::Matrix3d) is an inline
    overload that honours the row step and create()s the output; compiled against a cv::Mat stand-in with pixels and the Eigen stand-in of
    oracle/ref_shim.  With a GPU its result equals the restatement; without one it throws std::runtime_error (no CPU fallback)."""
    from line3dpp_b200 import build
    so = build.build()
    (tmp_path / "opencv2").mkdir()
    (tmp_path / "opencv2" / "core.hpp").write_text(MAT_STANDIN)
    src = tmp_path / "undist.cpp"
    src.write_text(FACADE)
    exe = tmp_path / "undist"
    cmd = ["g++", "-std=c++17", "-Wall", "-Werror", str(src), "-I" + os.path.join(ROOT, "include"), "-I" + str(tmp_path),
           "-I" + os.path.join(ROOT, "oracle", "ref_shim"), "-L" + os.path.dirname(so), "-ll3d_b200", "-Wl,-rpath," + os.path.dirname(so), "-o", str(exe)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = tmp_path / "out.raw"
    r = subprocess.run([str(exe), str(out)], capture_output=True, text=True)
    import torch
    if not torch.cuda.is_available():
        assert r.returncode == 3 and "no GPU" in r.stdout, (r.returncode, r.stdout)
        return
    assert r.returncode == 0, (r.returncode, r.stdout)
    y, x, c = np.meshgrid(np.arange(23), np.arange(37), np.arange(3), indexing="ij")
    img = ((x * 7 + y * 13 + c * 29) & 255).astype(np.uint8)
    ref = um.remap(img, *um.undistort_maps(37, 23, 41.5, 40.25, 17.75, 11.5, -0.21, 0.04, 0.01, 0.003, -0.002))
    assert np.array_equal(np.fromfile(out, np.uint8).reshape(23, 37, 3), ref)
