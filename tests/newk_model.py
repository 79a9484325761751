"""numpy restatement of the undistortion into a new camera matrix and size (l3d_undistort.cu with l3d_undistort_desc's new_fx ..
out_height; DESIGN.md §4a): OpenCV's initUndistortRectifyMap(K, D, I, newK, newSize) and cv::fisheye's with P = newK.  The output pixel
(j, i) goes back through the cofactor inverse of newK, and is distorted and projected with K, by the formulas of tests/undistort_model.py
and tests/lens_model.py.  TEST INFRASTRUCTURE, IEEE double without fused multiply-adds."""
import numpy as np

from tests import lens_model as lm
from tests import undistort_model as um


def radtan_uv(ow, oh, K, newK, k, p):
    """(iu, iv) int64 [oh, ow]: OpenCV's 8-coefficient model (k = k1..k6, p = p1, p2) into newK"""
    fx, fy, cx, cy = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
    k1, k2, k3, k4, k5, k6 = (float(v) for v in k)
    p1, p2 = float(p[0]), float(p[1])
    ir0, ir2, ir4, ir5 = um.inverse_k(float(newK[0, 0]), float(newK[1, 1]), float(newK[0, 2]), float(newK[1, 2]))
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        x = (np.arange(ow, dtype=np.float64) * ir0 + ir2)[None, :]
        y = (np.arange(oh, dtype=np.float64) * ir4 + ir5)[:, None]
        x2, y2 = x * x, y * y
        r2 = x2 + y2
        _2xy = 2.0 * x * y
        kr = (1.0 + ((k3 * r2 + k2) * r2 + k1) * r2) / (1.0 + ((k6 * r2 + k5) * r2 + k4) * r2)
        xd = x * kr + p1 * _2xy + p2 * (r2 + 2.0 * x2)
        yd = y * kr + p1 * (r2 + 2.0 * y2) + p2 * _2xy
        return um.fix32(fx * xd + cx), um.fix32(fy * yd + cy)


def fisheye_uv(ow, oh, K, newK, k):
    """(iu, iv) int64 [oh, ow]: cv::fisheye's model (k = k1..k4) into newK; x accumulated along the row from newK's (ir0, ir2)"""
    fx, fy, cx, cy = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
    k1, k2, k3, k4 = (float(v) for v in k[:4])
    ir0, ir2, ir4, ir5 = um.inverse_k(float(newK[0, 0]), float(newK[1, 1]), float(newK[0, 2]), float(newK[1, 2]))
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        x = lm.fisheye_columns(ow, ir0, ir2)[None, :]
        y = (np.arange(oh, dtype=np.float64) * ir4 + ir5)[:, None]
        r = np.sqrt(x * x + y * y)
        th = np.arctan(r)
        t2 = th * th
        t4 = t2 * t2
        t6 = t4 * t2
        t8 = t4 * t4
        thd = th * (1.0 + k1 * t2 + k2 * t4 + k3 * t6 + k4 * t8)
        scale = np.where(r == 0.0, 1.0, thd / np.where(r == 0.0, 1.0, r))
        return um.fix32(fx * x * scale + cx), um.fix32(fy * y * scale + cy)


def newk_maps(ow, oh, K, newK, model, k, p):
    """map_xy int16 [oh, ow, 2], map_frac uint16 [oh, ow]; k = k1..k6 (radtan) or k1..k4 (fisheye), p = p1, p2"""
    k = [float(v) for v in k] + [0.0] * (6 - len(k))
    if model == lm.FISHEYE:
        return lm.maps_wrapped(*fisheye_uv(ow, oh, K, newK, k))
    return um.maps_from_uv(*radtan_uv(ow, oh, K, newK, k, p))


def case_params(g, name):
    """(w, h, c, K, model, k[6], p[2], newK, (ow, oh)) of one case of tests/golden/ref_undistort_newk_v1.npz"""
    s, o = g[f"{name}/size"], g[f"{name}/out_size"]
    return (int(s[0]), int(s[1]), int(s[2]), g[f"{name}/K"], int(g[f"{name}/model"]), g[f"{name}/k"], g[f"{name}/p"], g[f"{name}/cv_newK"],
            (int(o[0]), int(o[1])))


def lens_dict(model, k, p):
    """the lens dict of line3d.read_colmap for the parameters of a case"""
    return {"model": int(model), "k": np.asarray(k, np.float64), "p": np.asarray(p, np.float64)}
