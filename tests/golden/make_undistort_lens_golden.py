"""Writes tests/golden/ref_undistort_lens_v1.npz: what OpenCV computes for the two lens models l3d_undistort.cu adds (DESIGN.md §4a):
cv::fisheye::initUndistortRectifyMap(K, D, I, K) and the 8-coefficient cv::initUndistortRectifyMap(K, D, I, K), both with CV_16SC2 +
CV_16UC1 maps, then remap INTER_LINEAR / BORDER_CONSTANT 0.  K is passed without skew, as the reference does.

Needs cv2 (any CPU machine).  Same layout as ref_undistort_v1.npz (make_undistort_golden.py); per case:
  <name>/size, /K, /model, /k, /p                  parameters (model 0 radtan: k = k1..k6; model 1 fisheye: k = k1..k4, 0, 0; p = p1, p2)
  <name>/cv_map_sha                                SHA-256 of cv2's map1 (int16 [h, w, 2]) followed by map2 (uint16 [h, w])
  <name>/diff_idx, /diff_xy, /diff_frac            flat pixel index and cv2's entry wherever cv2's maps differ from tests/lens_model.py's
  <name>/cv_remap_sha, /model_remap_sha            SHA-256 of cv2.remap with cv2's maps, resp. with the model's maps
and cv2_version / cv2_cpu.

    python tests/golden/make_undistort_lens_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests import lens_model as lm  # noqa: E402
from tests import undistort_model as um  # noqa: E402
from tests.golden.make_undistort_golden import cpu_features  # noqa: E402

OUT = os.path.join(HERE, "ref_undistort_lens_v1.npz")
F, R = lm.FISHEYE, lm.RADTAN

# name: (w, h, channels, (fx, fy, cx, cy), model, k, p)
CASES = {
    "fisheye": (3072, 2304, 1, (1100.0, 1100.0, 1536.0, 1152.0), F, (0.05, -0.01, 0.003, -0.0005), (0, 0)),       # OPENCV_FISHEYE
    "fisheye_k": (1600, 1200, 3, (700.0, 700.0, 800.0, 600.0), F, (0.08, 0, 0, 0), (0, 0)),                     # SIMPLE_RADIAL_FISHEYE
    "fisheye_k1k2": (1280, 960, 3, (610.5, 610.5, 640.0, 480.0), F, (0.07, -0.02, 0, 0), (0, 0)),               # RADIAL_FISHEYE
    "fisheye_strong": (1280, 960, 1, (420.0, 420.0, 640.0, 480.0), F, (0.4, 0.2, 0.05, 0.01), (0, 0)),           # map leaves the image
    "fisheye_int16": (3072, 2304, 1, (1000.0, 1000.0, 1536.0, 1152.0), F, (40.0, 0, 0, 0), (0, 0)),             # u, v leave int16
    "fisheye_odd": (1001, 777, 3, (905.25, 921.6, 487.3, 401.9), F, (0.02, 0.01, -0.004, 0.001), (0, 0)),      # odd size, fx != fy
    "rational": (3072, 2304, 1, (2800.0, 2800.0, 1536.0, 1152.0), R, (0.12, -0.05, 0.01, 0.08, -0.02, 0.005), (0.0007, -0.0004)),
    "rational_odd": (1001, 777, 3, (905.25, 921.6, 487.3, 401.9), R, (-0.3, 0.1, -0.01, -0.25, 0.06, -0.002), (0.0012, -0.0021)),
    "rational_zero": (1001, 777, 3, (905.25, 921.6, 487.3, 401.9), R, (0.1, -0.05, 0.02, 0, 0, 0), (0.0012, -0.0021)),  # k4..k6 = 0
}


def cv_maps(cv2, w, h, fx, fy, cx, cy, model, k, p):
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float64)
    if model == F:
        return cv2.fisheye.initUndistortRectifyMap(K, np.array(k[:4], np.float64), np.eye(3), K, (w, h), cv2.CV_16SC2)
    dist = np.array([k[0], k[1], p[0], p[1], k[2], k[3], k[4], k[5]], np.float64)
    return cv2.initUndistortRectifyMap(K, dist, np.eye(3), K, (w, h), cv2.CV_16SC2)


def main():
    import cv2
    out = {"cv2_version": np.array(cv2.__version__), "cv2_cpu": np.array(cpu_features(cv2)), "cases": np.array(list(CASES))}
    for i, (name, (w, h, c, (fx, fy, cx, cy), model, k, p)) in enumerate(CASES.items()):
        k = tuple(float(v) for v in k) + (0.0,) * (6 - len(k))
        m1, m2 = cv_maps(cv2, w, h, fx, fy, cx, cy, model, k, p)
        xy, fr = lm.lens_maps(w, h, fx, fy, cx, cy, model, k, p)
        diff = np.flatnonzero((m1.reshape(-1, 2) != xy.reshape(-1, 2)).any(axis=1) | (m2.reshape(-1) != fr.reshape(-1)))
        img = um.make_image(h, w, c, seed=100 + i)
        P = f"{name}/"
        out[P + "size"] = np.array([w, h, c], np.int64)
        out[P + "K"] = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float64)
        out[P + "model"] = np.array(model, np.int64)
        out[P + "k"], out[P + "p"] = np.array(k, np.float64), np.array(p, np.float64)
        out[P + "cv_map_sha"] = np.array(um.sha(m1, m2))
        out[P + "diff_idx"] = diff.astype(np.int64)
        out[P + "diff_xy"] = m1.reshape(-1, 2)[diff]
        out[P + "diff_frac"] = m2.reshape(-1)[diff]
        out[P + "cv_remap_sha"] = np.array(um.sha(cv2.remap(img, m1, m2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)))
        out[P + "model_remap_sha"] = np.array(um.sha(cv2.remap(img, xy, fr, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)))
        print(f"{name:15s} {w}x{h}x{c}: {len(diff)} map entries differ from the model")
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes;", out["cv2_version"], out["cv2_cpu"])


if __name__ == "__main__":
    main()
