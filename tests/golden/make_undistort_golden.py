"""Writes tests/golden/ref_undistort_v1.npz: what OpenCV computes for Line3D::undistortImage (line3D.cc:83-109:
initUndistortRectifyMap with CV_16SC2 + CV_16UC1 maps, remap INTER_LINEAR / BORDER_CONSTANT 0) on the cases below.

Needs cv2 (any CPU machine).  The input images come from tests/undistort_model.make_image (integer hash), so nothing but digests and
the few map entries where OpenCV's accumulation order differs from the model's formula is stored.  Per case:
  <name>/size, /K, /radial, /tangential     parameters (K may carry a skew; like the reference, only fx, fy, cx, cy are used)
  <name>/cv_map_sha                          SHA-256 of cv2's map1 (int16 [h, w, 2]) followed by map2 (uint16 [h, w])
  <name>/diff_idx, /diff_xy, /diff_frac      flat pixel index and cv2's entry wherever cv2's maps differ from the model's
  <name>/cv_remap_sha                        SHA-256 of cv2.remap with cv2's maps
  <name>/model_remap_sha                     SHA-256 of cv2.remap with the model's maps
and cv2_version / cv2_cpu (baseline and dispatched CPU features of that build).

    python tests/golden/make_undistort_golden.py
"""
import os
import re
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests import undistort_model as um  # noqa: E402

OUT = os.path.join(HERE, "ref_undistort_v1.npz")

# name: (w, h, channels, K, radial (k1, k2, k3), tangential (p1, p2))
CASES = {
    "vsfm": (3072, 2304, 1, [[2800.0, 0, 1536.0], [0, 2800.0, 1152.0], [0, 0, 1]], (-0.08, 0, 0), (0, 0)),            # VisualSfM: (-d, 0, 0)
    "bundler": (1600, 1200, 3, [[1350.5, 0, 800.0], [0, 1350.5, 600.0], [0, 0, 1]], (-0.12, 0.05, 0), (0, 0)),        # Bundler: k1, k2
    "colmap_opencv": (1001, 777, 3, [[905.25, 1.75, 487.3], [0, 921.6, 401.9], [0, 0, 1]], (0.1, -0.05, 0.02),       # odd size, fx != fy,
                      (0.0012, -0.0021)),                                                                             # skew (ignored), k3
    "zero": (640, 480, 3, [[500.0, 0, 320.0], [0, 500.0, 240.0], [0, 0, 1]], (0, 0, 0), (0, 0)),                     # identity
    "k1_20": (3072, 2304, 1, [[2800.0, 0, 1536.0], [0, 2800.0, 1152.0], [0, 0, 1]], (20.0, 0, 0), (0, 0)),          # int16 saturation
    "k1_m3": (1024, 768, 1, [[700.0, 0, 512.0], [0, 700.0, 384.0], [0, 0, 1]], (-3.0, 0, 0), (0, 0)),               # map folds back
    "tiny": (17, 13, 3, [[20.0, 0, 7.5], [0, 22.0, 6.25], [0, 0, 1]], (0.2, 0, 0), (0.01, 0)),
}


def cpu_features(cv2):
    info = cv2.getBuildInformation()
    lines = [m.group(0).strip() for m in re.finditer(r"^\s*(Baseline|Dispatched code generation):.*$", info, re.M)]
    return " | ".join(lines)


def main():
    import cv2
    out = {"cv2_version": np.array(cv2.__version__), "cv2_cpu": np.array(cpu_features(cv2)), "cases": np.array(list(CASES))}
    for i, (name, (w, h, c, K, rad, tan)) in enumerate(CASES.items()):
        K = np.array(K, np.float64)
        cvK = np.array([[K[0, 0], 0, K[0, 2]], [0, K[1, 1], K[1, 2]], [0, 0, 1]], np.float64)        # line3D.cc:88-93
        dist = np.array([rad[0], rad[1], tan[0], tan[1], rad[2]], np.float64)
        m1, m2 = cv2.initUndistortRectifyMap(cvK, dist, np.eye(3), cvK, (w, h), cv2.CV_16SC2)
        xy, fr = um.undistort_maps(w, h, K[0, 0], K[1, 1], K[0, 2], K[1, 2], rad[0], rad[1], rad[2], tan[0], tan[1])
        diff = np.flatnonzero((m1.reshape(-1, 2) != xy.reshape(-1, 2)).any(axis=1) | (m2.reshape(-1) != fr.reshape(-1)))
        img = um.make_image(h, w, c, seed=i)
        P = f"{name}/"
        out[P + "size"] = np.array([w, h, c], np.int64)
        out[P + "K"], out[P + "radial"], out[P + "tangential"] = K, np.array(rad, np.float64), np.array(tan, np.float64)
        out[P + "cv_map_sha"] = np.array(um.sha(m1, m2))
        out[P + "diff_idx"] = diff.astype(np.int64)
        out[P + "diff_xy"] = m1.reshape(-1, 2)[diff]
        out[P + "diff_frac"] = m2.reshape(-1)[diff]
        out[P + "cv_remap_sha"] = np.array(um.sha(cv2.remap(img, m1, m2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)))
        out[P + "model_remap_sha"] = np.array(um.sha(cv2.remap(img, xy, fr, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)))
        print(f"{name:14s} {w}x{h}x{c}: {len(diff)} map entries differ from the model")
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes;", out["cv2_version"], out["cv2_cpu"])


if __name__ == "__main__":
    main()
