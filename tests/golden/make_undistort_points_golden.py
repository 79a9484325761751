"""Writes tests/golden/ref_undistort_points_v1.npz: what OpenCV 4.13 returns for the point undistortion l3d_undistort_points restates
(DESIGN.md §4a): cv2.undistortPoints(src, K, D, None, P) for radtan lenses (5 and 8 coefficients) and cv2.fisheye.undistortPoints(src, K,
D, R=I, P=P) for fisheye lenses, float32 points, P = K or a new camera matrix (from cv2.getOptimalNewCameraMatrix /
cv2.fisheye.estimateNewCameraMatrixForUndistortRectify).  The points of every case: a dense grid over and far beyond the image, the
principal point and points within 1e-8 (normalised) of it, NaN and +-inf coordinates; the radtan and fisheye cases with strong lenses
reach the icdist < 0 fallback, fisheye non-convergence and theta flips (their counts are stored).  The "nvm" cases: the segment endpoints
of tests/golden/nvm_inputs_v1.npz (detected in the raw photos of the reference's testdata) under each camera's NVM radial lens, D = (-d, 0,
0, 0, 0) as the reference's VisualSfM frontend passes it to undistortImage (its first NVM_CAMS cameras).

Before writing, every case is checked: tests/undistort_points_model.py must give cv2's output bit for bit (NaN as NaN).

Needs cv2.  Per case:
  <name>/K, /new_K (3x3; new_K all zero: K), /model (0 radtan, 1 fisheye), /k (6: k1..k6, or k1..k4, 0, 0), /p (2)
  <name>/pts, /cv                              float32 [n, 2]: the input points and cv2's output
  <name>/fallback, /unconverged, /flipped      how many points take those paths (from the model)
and cases, cv2_version.

    python tests/golden/make_undistort_points_golden.py
"""
import gzip
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests import undistort_points_model as m  # noqa: E402

OUT = os.path.join(HERE, "ref_undistort_points_v1.npz")
R, F = m.RADTAN, m.FISHEYE
W, H = 3072, 2304
NVM_CAMS = 3        # the first cameras of the NVM model: ~8k segments


def kmat(fx, fy, cx, cy):
    return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float64)


def test_points(K, rng):
    """grid over and beyond the image, the principal point and its float32 neighbours, random far points, non-finite values"""
    gx, gy = np.meshgrid(np.linspace(-1.5 * W, 2.5 * W, 61), np.linspace(-1.5 * H, 2.5 * H, 46))
    grid = np.stack([gx.ravel(), gy.ravel()], 1)
    inner = np.stack(np.meshgrid(np.arange(0, W + 1, 128.0) + 0.25, np.arange(0, H + 1, 128.0) + 0.5), -1).reshape(-1, 2)
    cx, cy = np.float32(K[0, 2]), np.float32(K[1, 2])
    near = []
    for i in range(-3, 4):
        for j in range(-3, 4):
            x = cx
            y = cy
            for _ in range(abs(i)):
                x = np.nextafter(x, np.float32(np.inf * np.sign(i)))
            for _ in range(abs(j)):
                y = np.nextafter(y, np.float32(np.inf * np.sign(j)))
            near.append((x, y))
    far = rng.normal(0, 4 * W, (500, 2))
    special = [(np.nan, 100), (100, np.nan), (np.nan, np.nan), (np.inf, 100), (-np.inf, 100), (100, np.inf), (100, -np.inf),
               (np.inf, -np.inf), (1e30, 1e30), (-3e38, 5), (-5000, 9000), (0, 0), (W, H)]
    return np.concatenate([grid, inner, np.array(near, np.float64), far, np.array(special, np.float64)]).astype(np.float32)


def cases(cv2):
    rng = np.random.default_rng(7)
    K1 = kmat(2400.0, 2410.0, 1530.5, 1160.25)
    K2 = kmat(1100.0, 1100.0, 1536.0, 1152.0)
    K3 = kmat(905.25, 921.6, 1487.3, 1101.9)
    r5 = ((-0.12, 0.05, 0.0, 0, 0, 0), (0.001, -0.0007))
    r8 = ((0.12, -0.05, 0.01, 0.08, -0.02, 0.005), (0.0007, -0.0004))
    r8s = ((-0.3, 0.1, -0.01, -0.25, 0.06, -0.002), (0.0012, -0.0021))      # the fallback on most far points
    f4 = (0.05, -0.01, 0.003, -0.0005)
    fs = (-0.3, 0.0, 0.0, 0.0)                                               # non-convergence and theta flips
    D = lambda k, p: np.array([k[0], k[1], p[0], p[1], k[2]] + ([k[3], k[4], k[5]] if any(k[3:]) else []), np.float64)
    opt5, _ = cv2.getOptimalNewCameraMatrix(K1, D(*r5), (W, H), 0.5, (W, H))
    opt8, _ = cv2.getOptimalNewCameraMatrix(K3, D(*r8), (W, H), 1.0, (W, H))
    fnew = cv2.fisheye.estimateNewCameraMatrixForUndistortRectify(K2, np.array(f4), (W, H), np.eye(3), balance=0.5)
    out = {
        "radtan5": (K1, None, R, r5[0], r5[1]),
        "radtan5_opt": (K1, opt5, R, r5[0], r5[1]),
        "radtan8": (K3, None, R, r8[0], r8[1]),
        "radtan8_opt": (K3, opt8, R, r8[0], r8[1]),
        "radtan8_fallback": (K1, kmat(1800.0, 1810.0, 1500.0, 1100.0), R, r8s[0], r8s[1]),
        "fisheye": (K2, None, F, f4 + (0, 0), (0, 0)),
        "fisheye_new": (K2, fnew, F, f4 + (0, 0), (0, 0)),
        "fisheye_fail": (K3, None, F, fs + (0, 0), (0, 0)),
    }
    res = {name: (c, test_points(c[0], rng)) for name, c in out.items()}
    # the reference's segments under the NVM radial lens
    nvm = np.load(os.path.join(HERE, "nvm_inputs_v1.npz"))
    lines = gzip.open(os.path.join(HERE, "vsfm_result_head.nvm.gz"), "rt").read().split("\n")
    dist = {ln.split()[0]: float(np.float32(ln.split()[9])) for ln in lines[3:3 + int(lines[2].split()[0])]}
    for i in range(NVM_CAMS):
        d = dist[str(nvm["names"][i])]
        res[f"nvm_{i}"] = ((nvm["K"][i], None, R, (-d, 0, 0, 0, 0, 0), (0, 0)), nvm[f"segs_{i}"].astype(np.float32).reshape(-1, 2))
    return res


def main():
    import cv2
    out = {"cv2_version": np.array(cv2.__version__)}
    names = []
    for name, ((K, nK, model, k, p), pts) in cases(cv2).items():
        k = tuple(float(v) for v in k)
        cv = m.cv2_undistort_points(cv2, pts, K, model, k, p, nK)
        info = {}
        mod = m.undistort_points(pts, K, model, k, p, nK, info=info)
        assert m.same(cv, mod), f"{name}: the model differs from cv2 at {np.flatnonzero(~((cv == mod) | (np.isnan(cv) & np.isnan(mod))).all(1))[:10]}"
        P = f"{name}/"
        out[P + "K"] = np.asarray(K, np.float64)
        out[P + "new_K"] = np.zeros((3, 3)) if nK is None else np.asarray(nK, np.float64)
        out[P + "model"] = np.array(model)
        out[P + "k"] = np.array(k, np.float64)
        out[P + "p"] = np.array(p, np.float64)
        out[P + "pts"] = pts
        out[P + "cv"] = cv
        for key in ("fallback", "unconverged", "flipped"):
            out[P + key] = np.array(int(info[key].sum()) if key in info else 0)
        names.append(name)
        print(f"{name}: {len(pts)} points, " + ", ".join(f"{key} {int(out[P + key])}" for key in ("fallback", "unconverged", "flipped")))
    out["cases"] = np.array(names)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
