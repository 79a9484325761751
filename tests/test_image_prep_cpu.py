"""Image preparation for line detection without a GPU: the numpy restatement (tests/image_prep_model.py) against what OpenCV computed
(tests/golden/ref_image_prep_v1.npz, tests/golden/make_image_prep_golden.py); detectLineSegments' post-processing in the restatement, in
the library (l3dpp_filter_detections) and in a std::priority_queue program; and the image overloads of include/line3d.h compiled
against header stand-ins."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from tests import image_prep_model as pm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_image_prep_v1.npz")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLDEN)


def _cases():
    return [str(n) for n in np.load(GOLDEN)["cases"]]


def case_image(g, name):
    """(image, max_img_width, row padding) of a golden case"""
    w, h, c, mw, seed, pad = (int(v) for v in g[f"{name}/params"])
    return pm.make_image(h, w, c, seed=seed), mw, pad


@pytest.mark.parametrize("name", _cases())
def test_model_reproduces_opencv(gold, name):
    img, mw, _ = case_image(gold, name)
    out = pm.prepare(img, mw)
    assert [out.shape[1], out.shape[0]] == gold[f"{name}/out_size"].tolist()
    assert pm.sha(out) == str(gold[f"{name}/cv_sha"])
    if f"{name}/cv_out" in gold:
        assert np.array_equal(out, gold[f"{name}/cv_out"])


def test_gray_table_sample(gold):
    rgb = gold["gray_rgb"]
    assert np.array_equal(pm.gray(rgb.reshape(-1, 1, 3)).reshape(-1), gold["gray_val"])


def test_cases_reach_every_branch(gold):
    modes = set()
    for name in _cases():
        w, h, c, mw, _, pad = (int(v) for v in gold[f"{name}/params"])
        ow, oh, resized = pm.prepared_size(w, h, mw)
        modes.add(("area2" if pm.scale_of(w, h, mw) == 2.0 else "linear") if resized else "copy")
        modes.add(("channels", c))
        modes.add("padded" if pad else "packed")
        modes.add("portrait" if h > w else "landscape")
        if resized and pm.scale_of(w, h, mw) in (3.0, 4.0):
            modes.add("integer step")
        if ow % 8:
            modes.add("width not a multiple of 8")
    assert modes >= {"copy", "area2", "linear", ("channels", 1), ("channels", 3), "padded", "packed", "portrait", "landscape",
                     "integer step", "width not a multiple of 8"}


def test_prep_size_is_the_segment_cache_rounding():
    """l3d_image_prep_size and the segment cache's file name share one rounding (preparedImageSize); the model agrees"""
    from line3dpp_b200 import capi, line3d
    rng = np.random.default_rng(3)
    sizes = [(3072, 2304, 1920), (2304, 3072, 1920), (3072, 2304, 1536), (401, 300, 256), (1000, 800, -1), (1000, 800, 1000), (1, 1, 0)]
    sizes += [(int(a), int(b), int(m)) for a, b, m in zip(rng.integers(1, 8000, 300), rng.integers(1, 8000, 300), rng.integers(-5, 6000, 300))]
    for w, h, mw in sizes:
        ow, oh, resized = capi.image_prep_size(w, h, mw)
        assert (ow, oh, resized) == pm.prepared_size(w, h, mw), (w, h, mw)
        assert line3d.segment_cache_path("/f", 3, w, h, mw) == f"/f/L3D++_data/segments_L3D++_3_{ow}x{oh}_3000.bin"
    L = capi.lib()
    o = C.c_int32()
    for bad in ((0, 5, -1), (5, 0, -1), (32768, 5, -1), (5, 40000, 100)):
        assert L.l3d_image_prep_size(*bad, C.byref(o), C.byref(o)) == -1
    assert L.l3d_image_prep_size(5, 5, -1, None, C.byref(o)) == -1


# ------------------------------------------------------------------------------------------------ post-processing
PQ_PROGRAM = r"""
// detectLineSegments' post-processing (line3D.cc:320-360) around std::priority_queue, with SegmentData2D and its comparison
// (commons.h:135-156) restated; reads w h w_p h_p max_segments n and n*4 floats from stdin, writes the kept floats to stdout
#include <cmath>
#include <cstdio>
#include <queue>
#include <vector>
struct SegmentData2D { float p1x_, p1y_, p2x_, p2y_, length_; };
struct SegmentData2D_comparison { bool operator()(const SegmentData2D& l, const SegmentData2D& r) const { return l.length_ < r.length_; } };
int main() {
    int w, h, wp, hp; unsigned int max_segments; long n;
    if (std::fread(&w, 4, 1, stdin) != 1 || std::fread(&h, 4, 1, stdin) != 1 || std::fread(&wp, 4, 1, stdin) != 1 || std::fread(&hp, 4, 1, stdin) != 1 ||
        std::fread(&max_segments, 4, 1, stdin) != 1 || std::fread(&n, 8, 1, stdin) != 1) return 2;
    std::vector<float> d(4 * n);
    if (n && std::fread(d.data(), 4, 4 * n, stdin) != (size_t)(4 * n)) return 2;
    const float upscale_x = float(w) / float(wp), upscale_y = float(h) / float(hp);
    const float min_len = sqrtf(float(h * h) + float(w * w)) * 0.005f;
    std::priority_queue<SegmentData2D, std::vector<SegmentData2D>, SegmentData2D_comparison> sorted;
    for (long i = 0; i < n; ++i) {
        SegmentData2D s;
        s.p1x_ = d[4 * i] * upscale_x; s.p1y_ = d[4 * i + 1] * upscale_y; s.p2x_ = d[4 * i + 2] * upscale_x; s.p2y_ = d[4 * i + 3] * upscale_y;
        float dx = s.p1x_ - s.p2x_, dy = s.p1y_ - s.p2y_;
        s.length_ = sqrtf(dx * dx + dy * dy);
        if (s.length_ > min_len) sorted.push(s);
    }
    const unsigned int keep = sorted.size() < max_segments ? (unsigned int)sorted.size() : max_segments;
    for (unsigned int pos = 0; !sorted.empty() && pos < keep; ++pos) {
        const SegmentData2D s = sorted.top();
        const float o[4] = {s.p1x_, s.p1y_, s.p2x_, s.p2y_};
        std::fwrite(o, 4, 4, stdout);
        sorted.pop();
    }
    return 0;
}
"""


def detection_sets():
    """(name, detections float32 [n, 4], w, h, w_p, h_p, max_segments)"""
    rng = np.random.default_rng(11)
    out = []
    # equal lengths in many directions: the pop order of ties is the heap's
    base = rng.uniform(0, 700, (64, 2)).astype(np.float32)
    eq = []
    for k, (x, y) in enumerate(base):
        L = np.float32([60, 60, 200, 35][k % 4])
        v = np.float32([3, 4, 0, 5][k % 4]), np.float32([4, 3, 5, 0][k % 4])      # |v| = 5 exactly: four directions, equal lengths
        eq.append([x, y, x + v[0] * L / 5, y + v[1] * L / 5])
    out.append(("equal lengths", np.array(eq, np.float32), 1000, 800, 1000, 800, 3000))
    # just below, at and above the threshold (no resize, so lengths are exact)
    w, h = 1000, 800
    m = np.float32(np.sqrt(np.float32(h * h) + np.float32(w * w))) * np.float32(0.005)
    edge = [[10, 20, 10 + t, 20] for t in (np.nextafter(m, np.float32(0)), m, np.nextafter(m, np.float32(1e9)))]
    edge += [[400, 10, 400, 10 + t] for t in (np.nextafter(m, np.float32(0)), m, np.nextafter(m, np.float32(1e9)))]
    out.append(("threshold", np.array(edge, np.float32), w, h, w, h, 3000))
    # resized image: the threshold is measured on the original
    wp, hp = 1920, 1440
    mr = np.float32(np.sqrt(np.float32(2304 * 2304) + np.float32(3072 * 3072))) * np.float32(0.005)
    ux = np.float32(3072) / np.float32(wp)
    near = [[5, 5, 5 + t / ux, 5] for t in np.linspace(mr * 0.99, mr * 1.01, 41, dtype=np.float32)]
    rnd = rng.uniform(0, [wp, hp, wp, hp], (400, 4)).astype(np.float32)
    out.append(("resized", np.concatenate([np.array(near, np.float32), rnd]), 3072, 2304, wp, hp, 3000))
    # more than max_line_segments, with ties among them
    many = rng.uniform(0, 900, (700, 4)).astype(np.float32)
    many[::7] = many[1::7][: len(many[::7])]
    out.append(("cut", many, 1037, 811, 1000, 782, 100))
    out.append(("cut to one", many, 1037, 811, 1000, 782, 1))
    out.append(("none survive", np.array([[1, 1, 2, 2], [5, 5, 5, 6]], np.float32), 1000, 800, 1000, 800, 3000))
    out.append(("empty", np.zeros((0, 4), np.float32), 1000, 800, 1000, 800, 3000))
    return out


@pytest.fixture(scope="module")
def pq_exe(tmp_path_factory):
    d = tmp_path_factory.mktemp("pq")
    (d / "pq.cpp").write_text(PQ_PROGRAM)
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", str(d / "pq.cpp"), "-o", str(d / "pq")], check=True)
    return str(d / "pq")


@pytest.mark.parametrize("case", [c[0] for c in detection_sets()])
def test_postprocess_restatement_equals_priority_queue(pq_exe, case):
    from line3dpp_b200 import capi
    name, det, w, h, wp, hp, mx = next(c for c in detection_sets() if c[0] == case)
    stdin = np.array([w, h, wp, hp, mx], np.int32).tobytes() + np.array([len(det)], np.int64).tobytes() + det.tobytes()
    r = subprocess.run([pq_exe], input=stdin, capture_output=True, check=True)
    ref = np.frombuffer(r.stdout, np.float32).reshape(-1, 4)
    model = pm.postprocess(det, w, h, wp, hp, mx)
    assert model.tobytes() == ref.tobytes()
    L = capi.lib()
    lib_out = np.zeros((max(len(det), 1), 4), np.float32)
    n = L.l3dpp_filter_detections(det.ctypes.data_as(C.c_void_p), C.c_longlong(len(det)), w, h, wp, hp, C.c_uint(mx),
                                  lib_out.ctypes.data_as(C.c_void_p), C.c_longlong(len(lib_out)))
    assert lib_out[:n].tobytes() == ref.tobytes()
    if case == "equal lengths":
        lens = np.hypot(ref[:, 0] - ref[:, 2], ref[:, 1] - ref[:, 3])
        assert len(np.unique(lens)) < len(lens) and not np.array_equal(ref, det[np.argsort(-lens, kind="stable")])
    if case == "threshold":
        assert len(ref) == 2
    if case.startswith("cut"):
        assert len(ref) == mx


# ------------------------------------------------------------------------------------------------ the header's image overloads
MAT_STANDIN = r"""
// cv::Mat with pixels: the members include/line3d.h's addImage and undistortImage overloads use
#pragma once
#include <cstddef>
#include <vector>
#define CV_8UC1 0
#define CV_8UC3 16
#define CV_16UC1 2
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
    void create_padded(int r, int c, int t, size_t s) { rows = r; cols = c; type_ = t; step = s; buf_.assign(s * r, 0); data = buf_.data(); }
};
}  // namespace cv
"""

FACADE = r"""
#include "line3d.h"
#ifndef L3DPP_WITH_EIGEN_OPENCV
#error "the Eigen / OpenCV overloads were not enabled"
#endif
#include <cstdio>
#include <cstring>
#include <string>
// the prepared image it was given, and one segment across it
static bool detector(void* user, const L3DPP::Image8u& gray, std::vector<L3DPP::Vec4f>& out) {
    *(L3DPP::Image8u*)user = gray;
    L3DPP::Vec4f v = {{1.0f, 2.0f, float(gray.cols - 3), float(gray.rows - 4)}};
    out.push_back(v);
    return true;
}
int main(int argc, char** argv) {
    const bool pixels = argc > 2;
    try {
        L3DPP::Line3D L(argv[1], false, 500, 3000, false, true);
        L3DPP::Image8u seen;
        Eigen::Matrix3d K = Eigen::Matrix3d::Identity(), R = Eigen::Matrix3d::Identity();
        K(0, 0) = K(1, 1) = 900.0; K(0, 2) = 500.0; K(1, 2) = 400.0;
        Eigen::Vector3d t(0, 0, 1);
        std::list<unsigned int> nb(1, 7u);
        cv::Mat img;
#ifdef PIXELS
        img.create_padded(803, 1000, CV_8UC3, 3007);
        for (int y = 0; y < img.rows; ++y) for (int x = 0; x < 3 * img.cols; ++x) img.data[y * img.step + x] = (unsigned char)((x * 7 + y * 13) & 255);
#else
        img = cv::Mat(803, 1000, CV_8UC3);
#endif
        const bool without_detector = L.addImage(0u, img, K, R, t, 4.0f, nb);                    // rejected: no detector, no cache
        const std::string e0 = L.lastError();
        L.setSegmentDetector(detector, &seen);
        const bool with_detector = L.addImage(1u, img, K, R, t, 4.0f, nb);
        L3DPP::Image8u small(600, 700, 1);
        L3DPP::Matrix3d Kp, Rp;
        for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) { Kp(r, c) = K(r, c); Rp(r, c) = R(r, c); }
        const bool too_small = L.addImage(2u, small, Kp, Rp, L3DPP::Vector3d(0, 0, 1), 4.0f, nb);
        std::printf("%d %d %d %zu %dx%d | %s\n", int(without_detector), int(with_detector), int(too_small), L.numImages(), seen.cols, seen.rows, e0.c_str());
        if (pixels && argv[2][0]) {
            FILE* f = std::fopen(argv[2], "wb");
            std::fwrite(seen.data.data(), 1, seen.data.size(), f);
            std::fclose(f);
        }
        const bool want = pixels ? with_detector : !with_detector;     // without pixels the image cannot be prepared
        return (!without_detector && want && !too_small && e0.find("no line segments given") != std::string::npos) ? 0 : 1;
    } catch (const std::exception& e) { std::printf("no GPU: %s\n", e.what()); return 3; }
}
"""


@pytest.mark.parametrize("stand_in", ["ref_shim", "pixels"])
def test_image_overloads_compile_and_run(tmp_path, stand_in):
    """addImage(camID, cv::Mat&, ...) (the reference's signature), addImage(camID, const Image8u&, ...) and setSegmentDetector compile
    with -Wall -Wextra -Werror against the cv::Mat stand-in of oracle/ref_shim (no pixels) and one with pixels and a padded row step.
    With a GPU the pixel build prepares the image and calls the detector with it; the detector-less call is rejected with the
    unchanged message; without a GPU the constructor throws (no CPU fallback)."""
    from line3dpp_b200 import build
    so = build.build()
    inc = ["-I" + os.path.join(ROOT, "include")]
    if stand_in == "pixels":
        (tmp_path / "opencv2").mkdir()
        (tmp_path / "opencv2" / "core.hpp").write_text(MAT_STANDIN)
        inc += ["-I" + str(tmp_path), "-DPIXELS"]
    inc += ["-isystem", os.path.join(ROOT, "oracle", "ref_shim")]
    src = tmp_path / "facade.cpp"
    src.write_text(FACADE)
    exe = tmp_path / "facade"
    cmd = ["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", str(src)] + inc + ["-L" + os.path.dirname(so), "-ll3d_b200",
                                                                                  "-Wl,-rpath," + os.path.dirname(so), "-o", str(exe)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = tmp_path / "seen.raw"
    args = [str(exe), str(tmp_path)] + ([str(out)] if stand_in == "pixels" else [])
    r = subprocess.run(args, capture_output=True, text=True)
    import torch
    if not torch.cuda.is_available():
        assert r.returncode == 3 and "no GPU" in r.stdout, (r.returncode, r.stdout)
        return
    assert r.returncode == 0, (r.returncode, r.stdout)
    if stand_in == "pixels":
        y, x = np.meshgrid(np.arange(803), np.arange(3000), indexing="ij")
        img = ((x * 7 + y * 13) & 255).astype(np.uint8).reshape(803, 1000, 3)
        assert np.array_equal(np.fromfile(out, np.uint8).reshape(402, 500), pm.prepare(img, 500))
