"""Writes tests/golden/ref_undistort_newk_v1.npz: what OpenCV computes when it undistorts into a new camera matrix and size
(DESIGN.md §4a): cv2.getOptimalNewCameraMatrix / cv2.fisheye.estimateNewCameraMatrixForUndistortRectify for the new K, then
initUndistortRectifyMap(K, D, I, newK, newSize) (fisheye: cv2.fisheye's) with CV_16SC2 + CV_16UC1 maps and remap INTER_LINEAR /
BORDER_CONSTANT 0.  K is passed without skew.

Needs cv2 (any CPU machine).  The layout of ref_undistort_lens_v1.npz (make_undistort_lens_golden.py); per case:
  <name>/size, /K, /model, /k, /p                  source (w, h, c) and lens (model 0 radtan: k = k1..k6; 1 fisheye: k = k1..k4, 0, 0)
  <name>/out_size                                  the new size (w, h) the maps are built for
  <name>/alpha, /center, /new_size_arg             radtan: getOptimalNewCameraMatrix's alpha, centerPrincipalPoint and newImgSize
  <name>/balance, /fov_scale, /new_size_arg        fisheye: estimateNewCameraMatrixForUndistortRectify's arguments
  <name>/cv_newK, /cv_roi                          cv2's new camera matrix (3x3) and, radtan, validPixROI (x, y, w, h)
  <name>/cv_map_sha                                SHA-256 of cv2's map1 (int16 [oh, ow, 2]) followed by map2 (uint16 [oh, ow])
  <name>/diff_idx, /diff_xy, /diff_frac            flat pixel index and cv2's entry wherever cv2's maps differ from tests/newk_model.py's
  <name>/cv_remap_sha, /model_remap_sha            SHA-256 of cv2.remap with cv2's maps, resp. with the model's maps
and cv2_version / cv2_cpu.

    python tests/golden/make_undistort_newk_golden.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests import lens_model as lm  # noqa: E402
from tests import newk_model as nm  # noqa: E402
from tests import undistort_model as um  # noqa: E402
from tests.golden.make_undistort_golden import cpu_features  # noqa: E402

OUT = os.path.join(HERE, "ref_undistort_newk_v1.npz")
F, R = lm.FISHEYE, lm.RADTAN
R5 = (-0.25, 0.08, -0.01, 0, 0, 0), (0.001, -0.0007)
R8 = (0.12, -0.05, 0.01, 0.08, -0.02, 0.005), (0.0007, -0.0004)
# a lens that folds over: interior grid points undistort past the border's bounding box, which is all getOptimalNewCameraMatrix's
# outer rectangle bounds (an outer box over all 81 grid points gives another matrix and ROI)
RF = (-0.583, 0.52, -0.497, 0.414, -0.159, 0.541), (-0.002, 0.0087)
KR = (1000.0, 990.0, 640.5, 479.25)
KO = (905.25, 921.6, 487.3, 401.9)
FE = (0.05, -0.01, 0.002, -0.0005)

# name: (w, h, channels, (fx, fy, cx, cy), model, (k, p), arguments of the new-K function; new_size (0, 0): the source size)
CASES = {
    "radtan5_a0": (1280, 960, 1, KR, R, R5, dict(alpha=0.0, new_size=(0, 0), center=False)),
    "radtan5_a05_smaller": (1280, 960, 3, KR, R, R5, dict(alpha=0.5, new_size=(800, 600), center=False)),
    "radtan5_a1_larger": (1280, 960, 1, KR, R, R5, dict(alpha=1.0, new_size=(1600, 1200), center=False)),
    "radtan5_a05_center_nonprop": (1280, 960, 1, KR, R, R5, dict(alpha=0.5, new_size=(1500, 700), center=True)),
    "rational8_a0": (1001, 777, 3, KO, R, R8, dict(alpha=0.0, new_size=(0, 0), center=False)),
    "rational8_a05": (1001, 777, 1, KO, R, R8, dict(alpha=0.5, new_size=(0, 0), center=False)),
    "rational8_a1_nonprop": (1001, 777, 3, KO, R, R8, dict(alpha=1.0, new_size=(1400, 600), center=False)),
    "rational8_a1_center": (1001, 777, 1, KO, R, R8, dict(alpha=1.0, new_size=(0, 0), center=True)),
    "rational8_fold_a05": (1001, 777, 1, KO, R, RF, dict(alpha=0.5, new_size=(0, 0), center=False)),
    "rational8_fold_a1_center": (1001, 777, 3, KO, R, RF, dict(alpha=1.0, new_size=(0, 0), center=True)),
    "fisheye_b0": (3072, 2304, 1, (800.0, 800.0, 1536.0, 1152.0), F, (FE, (0, 0)), dict(balance=0.0, new_size=(0, 0), fov_scale=1.0)),
    "fisheye_b05_smaller": (1600, 1200, 3, (700.0, 690.0, 801.3, 598.7), F, (FE, (0, 0)), dict(balance=0.5, new_size=(1000, 750), fov_scale=1.0)),
    "fisheye_b1_larger_nonprop": (1280, 960, 1, (610.5, 610.5, 640.0, 480.0), F, ((0.07, -0.02, 0, 0), (0, 0)),
                                  dict(balance=1.0, new_size=(2000, 1100), fov_scale=1.0)),
    "fisheye_fov": (1001, 777, 3, KO, F, ((0.02, 0.01, -0.004, 0.001), (0, 0)), dict(balance=0.5, new_size=(0, 0), fov_scale=1.4)),
    "fisheye_int16": (3072, 2304, 1, (1000.0, 1000.0, 1536.0, 1152.0), F, ((40.0, 0, 0, 0), (0, 0)),
                      dict(balance=1.0, new_size=(0, 0), fov_scale=4.0)),   # u, v leave int16 under the new K
}


def cv_new_k(cv2, w, h, K, model, k, p, args):
    if model == F:
        P = cv2.fisheye.estimateNewCameraMatrixForUndistortRectify(K, np.array(k[:4], np.float64), (w, h), np.eye(3), balance=args["balance"],
                                                                   new_size=args["new_size"], fov_scale=args["fov_scale"])
        return P, np.zeros(4, np.int64)
    dist = np.array([k[0], k[1], p[0], p[1], k[2], k[3], k[4], k[5]], np.float64)
    M, roi = cv2.getOptimalNewCameraMatrix(K, dist, (w, h), args["alpha"], args["new_size"], centerPrincipalPoint=args["center"])
    return M, np.array(roi, np.int64)


def cv_maps(cv2, w, h, K, model, k, p, newK, out_size):
    if model == F:
        return cv2.fisheye.initUndistortRectifyMap(K, np.array(k[:4], np.float64), np.eye(3), newK, out_size, cv2.CV_16SC2)
    dist = np.array([k[0], k[1], p[0], p[1], k[2], k[3], k[4], k[5]], np.float64)
    return cv2.initUndistortRectifyMap(K, dist, np.eye(3), newK, out_size, cv2.CV_16SC2)


def main():
    import cv2
    out = {"cv2_version": np.array(cv2.__version__), "cv2_cpu": np.array(cpu_features(cv2)), "cases": np.array(list(CASES))}
    for i, (name, (w, h, c, (fx, fy, cx, cy), model, (k, p), args)) in enumerate(CASES.items()):
        k = tuple(float(v) for v in k) + (0.0,) * (6 - len(k))
        p = tuple(float(v) for v in p)
        K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float64)
        newK, roi = cv_new_k(cv2, w, h, K, model, k, p, args)
        ns = args["new_size"]
        out_size = (w, h) if ns[0] * ns[1] == 0 else ns
        m1, m2 = cv_maps(cv2, w, h, K, model, k, p, newK, out_size)
        xy, fr = nm.newk_maps(out_size[0], out_size[1], K, newK, model, k, p)
        diff = np.flatnonzero((m1.reshape(-1, 2) != xy.reshape(-1, 2)).any(axis=1) | (m2.reshape(-1) != fr.reshape(-1)))
        img = um.make_image(h, w, c, seed=200 + i)
        P = f"{name}/"
        out[P + "size"] = np.array([w, h, c], np.int64)
        out[P + "K"] = K
        out[P + "model"] = np.array(model, np.int64)
        out[P + "k"], out[P + "p"] = np.array(k, np.float64), np.array(p, np.float64)
        out[P + "out_size"] = np.array(out_size, np.int64)
        out[P + "new_size_arg"] = np.array(ns, np.int64)
        if model == F:
            out[P + "balance"], out[P + "fov_scale"] = np.array(args["balance"]), np.array(args["fov_scale"])
        else:
            out[P + "alpha"], out[P + "center"] = np.array(args["alpha"]), np.array(args["center"])
        out[P + "cv_newK"], out[P + "cv_roi"] = np.asarray(newK, np.float64), roi
        out[P + "cv_map_sha"] = np.array(um.sha(m1, m2))
        out[P + "diff_idx"] = diff.astype(np.int64)
        out[P + "diff_xy"] = m1.reshape(-1, 2)[diff]
        out[P + "diff_frac"] = m2.reshape(-1)[diff]
        out[P + "cv_remap_sha"] = np.array(um.sha(cv2.remap(img, m1, m2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)))
        out[P + "model_remap_sha"] = np.array(um.sha(cv2.remap(img, xy, fr, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)))
        print(f"{name:28s} {w}x{h}x{c} -> {out_size[0]}x{out_size[1]}: f' = {newK[0, 0]:.4f}, {len(diff)} map entries differ from the model")
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes;", out["cv2_version"], out["cv2_cpu"])


if __name__ == "__main__":
    main()
