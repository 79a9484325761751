"""The point undistortion contract without a GPU: the numpy restatement (tests/undistort_points_model.py) against what OpenCV computed
(tests/golden/ref_undistort_points_v1.npz), and the C++ surface of the feature (Line3D::undistortPoints / undistortSegments, the cv::Vec4f
overload, addImage with a lens) compiled against the public headers and the Eigen / OpenCV stand-ins of oracle/ref_shim."""
import os
import subprocess

import numpy as np
import pytest

from tests import undistort_points_model as m

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_undistort_points_v1.npz")


def _cases():
    return [str(n) for n in np.load(GOLDEN)["cases"]]


@pytest.mark.parametrize("name", _cases())
def test_model_equals_opencv(name):
    g = np.load(GOLDEN)
    P = f"{name}/"
    out = m.undistort_points(g[P + "pts"], g[P + "K"], int(g[P + "model"]), g[P + "k"], g[P + "p"], g[P + "new_K"])
    assert m.same(out, g[P + "cv"])


def test_golden_reaches_every_path():
    """the golden points take the radtan fallback, the fisheye failure value (non-convergence and flips), the principal-point branch and
    NaN / inf, so that the GPU test sees each of them"""
    g = np.load(GOLDEN)
    names = _cases()
    assert str(g["cv2_version"]).startswith("4.13")
    assert sum(int(g[f"{n}/fallback"]) for n in names) > 100
    assert sum(int(g[f"{n}/unconverged"]) for n in names) > 100 and sum(int(g[f"{n}/flipped"]) for n in names) > 10
    for n in names:
        pts, cv = g[f"{n}/pts"], g[f"{n}/cv"]
        if n.startswith("nvm"):
            assert np.isfinite(cv).all()
            continue
        assert (~np.isfinite(pts)).any() and (np.isnan(cv).any() or int(g[f"{n}/unconverged"]))   # NaN in, NaN or the failure value out
        K, nK = g[f"{n}/K"], g[f"{n}/new_K"]
        P = nK if np.any(nK) else K
        at_pp = (pts[:, 0] == np.float32(K[0, 2])) & (pts[:, 1] == np.float32(K[1, 2]))
        assert at_pp.sum() == 1
        if int(g[f"{n}/model"]) == m.FISHEYE and not int(g[f"{n}/unconverged"]):
            # theta_d <= 1e-8: scale 0, the new principal point exactly
            assert cv[at_pp][0].tolist() == [np.float32(P[0, 2]), np.float32(P[1, 2])]


def test_cpp_surface_compiles_against_eigen_opencv_stand_ins(tmp_path):
    from line3dpp_b200 import build
    so = build.build()
    src = tmp_path / "points.cpp"
    src.write_text(r"""
#include "line3d.h"
#ifndef L3DPP_WITH_EIGEN_OPENCV
#error "the Eigen / OpenCV overloads were not enabled"
#endif
#include <cstdio>
int main() {
    L3DPP::LensDistortion lens = {L3DPP::LensDistortion::RADTAN, {-0.1, 0.01, 0, 0, 0, 0}, {0, 0}};
    L3DPP::Matrix3d K = L3DPP::Matrix3d();
    K(0, 0) = 1000; K(1, 1) = 1000; K(0, 2) = 800; K(1, 2) = 600; K(2, 2) = 1;
    Eigen::Matrix3d Ke = Eigen::Matrix3d::Identity();
    Ke(0, 0) = 1000; Ke(1, 1) = 1000; Ke(0, 2) = 800; Ke(1, 2) = 600;
    try {
        std::vector<float> xy(4, 100.f);
        L3DPP::Line3D::undistortPoints(xy, lens, K);
        std::vector<L3DPP::Vec4f> segs(1);
        L3DPP::Line3D::undistortSegments(segs, lens, K, K);
        std::vector<std::vector<float> > sets(2, xy);
        L3DPP::Line3D::undistortPoints(sets, std::vector<L3DPP::LensDistortion>(2, lens), std::vector<L3DPP::Matrix3d>(2, K));
        std::vector<cv::Vec4f> cvsegs(1, cv::Vec4f(1.f, 2.f, 300.f, 400.f));
        L3DPP::Line3D::undistortSegments(cvsegs, lens, Ke);
        L3DPP::Line3D L("/tmp", true, -1, 3000, false, true);
        std::list<unsigned int> nb(1, 1u);
        L3DPP::Image8u img(1200, 1600, 1);
        bool a = L.addImage(0u, img, K, K, L3DPP::Vector3d(0, 0, 1), 4.0f, nb, lens, segs);
        bool b = L.addImage(1u, 1600, 1200, K, K, L3DPP::Vector3d(0, 0, 1), 4.0f, nb, lens, segs);
        std::printf("%f %f %d %d\n", xy[0], cvsegs[0](0), int(a), int(b));
        return 0;
    } catch (const std::runtime_error& e) { std::printf("no GPU: %s\n", e.what()); return 3; }
}
""")
    exe = tmp_path / "points"
    shim = os.path.join(ROOT, "oracle", "ref_shim")
    cmd = ["g++", "-std=c++17", "-Wall", "-Werror", str(src), "-I" + os.path.join(ROOT, "include"), "-I" + shim, "-L" + os.path.dirname(so), "-ll3d_b200",
           "-Wl,-rpath," + os.path.dirname(so), "-o", str(exe)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    import torch
    assert r.returncode == (0 if torch.cuda.is_available() else 3), (r.returncode, r.stdout, r.stderr)
