"""numpy restatement of the two lens models l3d_undistort.cu adds to the pinhole contract of tests/undistort_model.py (DESIGN.md §4a):
OpenCV's 8-coefficient rational model (initUndistortRectifyMap with k4, k5, k6) and OpenCV's fisheye model
(cv::fisheye::initUndistortRectifyMap with R = I and newK = K).  TEST INFRASTRUCTURE, IEEE double without fused multiply-adds."""
import numpy as np

from tests import undistort_model as um

RADTAN, FISHEYE = 0, 1


def rational_uv(w, h, fx, fy, cx, cy, k1, k2, k3, p1, p2, k4, k5, k6):
    """(iu, iv) int64 [h, w] of the rational model: the pinhole formula with kr divided by 1 + ((k6 r2 + k5) r2 + k4) r2"""
    ir0, ir2, ir4, ir5 = um.inverse_k(fx, fy, cx, cy)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        x = (np.arange(w, dtype=np.float64) * ir0 + ir2)[None, :]
        y = (np.arange(h, dtype=np.float64) * ir4 + ir5)[:, None]
        x2, y2 = x * x, y * y
        r2 = x2 + y2
        _2xy = 2.0 * x * y
        kr = (1.0 + ((k3 * r2 + k2) * r2 + k1) * r2) / (1.0 + ((k6 * r2 + k5) * r2 + k4) * r2)
        xd = x * kr + p1 * _2xy + p2 * (r2 + 2.0 * x2)
        yd = y * kr + p1 * (r2 + 2.0 * y2) + p2 * _2xy
        return um.fix32(fx * xd + cx), um.fix32(fy * yd + cy)


def fisheye_columns(w, ir0, ir2):
    """x of every column as OpenCV's fisheye loop forms it: ir2, then ir0 added once per column, in order"""
    x = np.empty(w, np.float64)
    acc = ir2
    for j in range(w):
        x[j] = acc
        acc = acc + ir0
    return x


def fisheye_uv(w, h, fx, fy, cx, cy, k1, k2, k3, k4):
    """(iu, iv) int64 [h, w] of the fisheye model; x accumulated along the row, y = i * ir4 + ir5"""
    ir0, ir2, ir4, ir5 = um.inverse_k(fx, fy, cx, cy)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        x = fisheye_columns(w, ir0, ir2)[None, :]
        y = (np.arange(h, dtype=np.float64) * ir4 + ir5)[:, None]
        r = np.sqrt(x * x + y * y)
        th = np.arctan(r)
        t2 = th * th
        t4 = t2 * t2
        t6 = t4 * t2
        t8 = t4 * t4
        thd = th * (1.0 + k1 * t2 + k2 * t4 + k3 * t6 + k4 * t8)
        scale = np.where(r == 0.0, 1.0, thd / np.where(r == 0.0, 1.0, r))
        return um.fix32(fx * x * scale + cx), um.fix32(fy * y * scale + cy)


def maps_wrapped(iu, iv):
    """the fisheye loop's maps: (short)(iu >> 5) wraps to int16 where the pinhole path saturates"""
    xy = np.stack([(iu >> 5).astype(np.int64), (iv >> 5).astype(np.int64)], axis=-1)
    xy = ((xy + 32768) % 65536 - 32768).astype(np.int16)
    return xy, ((iv & 31) * 32 + (iu & 31)).astype(np.uint16)


def lens_maps(w, h, fx, fy, cx, cy, model, k, p):
    """map_xy int16 [h, w, 2], map_frac uint16 [h, w] of one camera; k = k1..k6 (radtan) or k1..k4 (fisheye), p = p1, p2"""
    k = [float(v) for v in k] + [0.0] * (6 - len(k))
    if model == FISHEYE:
        return maps_wrapped(*fisheye_uv(w, h, fx, fy, cx, cy, k[0], k[1], k[2], k[3]))
    return um.maps_from_uv(*rational_uv(w, h, fx, fy, cx, cy, k[0], k[1], k[2], float(p[0]), float(p[1]), k[3], k[4], k[5]))


def case_params(g, name):
    """(w, h, c, K 3x3, model, k[6], p[2]) of one case of tests/golden/ref_undistort_lens_v1.npz"""
    s = g[f"{name}/size"]
    return int(s[0]), int(s[1]), int(s[2]), g[f"{name}/K"], int(g[f"{name}/model"]), g[f"{name}/k"], g[f"{name}/p"]


def model_maps_for(w, h, K, model, k, p):
    return lens_maps(w, h, float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), model, k, p)
