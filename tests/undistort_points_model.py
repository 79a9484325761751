"""numpy restatement of l3d_undistort_points (DESIGN.md §4a): OpenCV 4.13's point undistortion of float32 (x, y) points into the pixels of a
new camera matrix P (the camera's K unless one is given).
  RADTAN:  cv::undistortPoints(src, dst, K, D, noArray(), P), i.e. cvUndistortPointsInternal with TermCriteria(COUNT, 5, 0.01): five
           fixed-point steps (the EPS test is off), the icdist < 0 fallback to the plain normalised point, the identity tilt and
           rectification products spelled out (they turn an infinite coordinate into NaN), then (float).
  FISHEYE: cv::fisheye::undistortPoints(src, dst, K, D, I, P) with its default TermCriteria(MAX_ITER + EPS, 10, 1e-8): the division by f,
           theta_d clamped to [-pi/2, pi/2] by std::max / std::min (NaN becomes -pi/2), Newton steps, scale = tan(theta) / theta_d
           (0 when theta_d <= 1e-8), the failure value -1e6 for a step that did not converge or a theta that flipped sign.
TEST INFRASTRUCTURE: IEEE double without fused multiply-adds, in OpenCV's operation order, vectorised over the points."""
import numpy as np

RADTAN, FISHEYE = 0, 1
FAIL = -1000000.0


def _err():
    return np.errstate(over="ignore", invalid="ignore", divide="ignore")


def _mv(r0, r1, r2, x, y):
    """row (r0, r1, r2) of a Matx33d times (x, y, 1) as cv::Matx's product sums it: ((0 + r0 x) + r1 y) + r2 * 1"""
    return ((0.0 + r0 * x) + r1 * y) + r2 * 1.0


def radtan(pts, fx, fy, cx, cy, k, p, P, info=None):
    """pts float32 [n, 2] -> float32 [n, 2]; k = k1..k6, p = p1, p2, P = (fx', fy', cx', cy'); info: a dict that receives the fallback mask"""
    k0, k1, k4, k5, k6, k7 = (float(v) for v in k)      # OpenCV's k[0], k[1], k[4], k[5], k[6], k[7]: k1, k2, k3, k4, k5, k6
    k2, k3 = float(p[0]), float(p[1])
    k8 = k9 = k10 = k11 = 0.0                            # thin prism terms: zero, but their products still run
    nfx, nfy, ncx, ncy = (float(v) for v in P)
    u = pts[:, 0].astype(np.float64)
    v = pts[:, 1].astype(np.float64)
    with _err():
        ifx, ify = 1.0 / fx, 1.0 / fy
        x = (u - cx) * ifx
        y = (v - cy) * ify
        ux = _mv(1.0, 0.0, 0.0, x, y)                  # invMatTilt = I
        uy = _mv(0.0, 1.0, 0.0, x, y)
        uz = _mv(0.0, 0.0, 1.0, x, y)
        inv = np.where(uz != 0, 1.0 / uz, 1.0)
        x0 = x = inv * ux
        y0 = y = inv * uy
        done = np.zeros(len(u), bool)
        for _ in range(5):
            r2 = x * x + y * y
            icdist = (1 + ((k7 * r2 + k6) * r2 + k5) * r2) / (1 + ((k4 * r2 + k1) * r2 + k0) * r2)
            fb = ~done & (icdist < 0)
            x = np.where(fb, (u - cx) * ifx, x)
            y = np.where(fb, (v - cy) * ify, y)
            done |= fb
            dx = 2 * k2 * x * y + k3 * (r2 + 2 * x * x) + k8 * r2 + k9 * r2 * r2
            dy = k2 * (r2 + 2 * y * y) + 2 * k3 * x * y + k10 * r2 + k11 * r2 * r2
            x = np.where(done, x, (x0 - dx) * icdist)
            y = np.where(done, y, (y0 - dy) * icdist)
        if info is not None:
            info["fallback"] = done
        # RR = P * I (cvMatMul): P's entries, zeros included
        xx = (nfx * x + 0.0 * y) + ncx
        yy = (0.0 * x + nfy * y) + ncy
        ww = 1.0 / ((0.0 * x + 0.0 * y) + 1.0)
        return np.stack([xx * ww, yy * ww], axis=1).astype(np.float32)


def fisheye(pts, fx, fy, cx, cy, k, P, tan=np.tan, info=None):
    """pts float32 [n, 2] -> float32 [n, 2]; k = k1..k4, P = (fx', fy', cx', cy'); tan: the tangent used (the host's by default); info: a
    dict that receives the masks of the points that did not converge and of those whose theta flipped"""
    k0, k1, k2, k3 = (float(v) for v in k[:4])
    nfx, nfy, ncx, ncy = (float(v) for v in P)
    u = pts[:, 0].astype(np.float64)
    v = pts[:, 1].astype(np.float64)
    with _err():
        pwx = (u - cx) / fx
        pwy = (v - cy) / fy
        td = np.sqrt(pwx * pwx + pwy * pwy)
        hp = np.pi / 2.0
        td = np.where(-hp < td, td, -hp)               # std::max(-pi/2, td) = (-pi/2 < td) ? td : -pi/2
        td = np.where(hp < td, hp, td)                 # std::min(td, pi/2) = (pi/2 < td) ? pi/2 : td
        newton = np.abs(td) > 1e-8
        theta = td.copy()
        conv = ~newton
        for _ in range(10):
            act = newton & ~conv
            t2 = theta * theta
            t4 = t2 * t2
            t6 = t4 * t2
            t8 = t6 * t2
            a, b, c, d = k0 * t2, k1 * t4, k2 * t6, k3 * t8
            fix = (theta * (1 + a + b + c + d) - td) / (1 + 3 * a + 5 * b + 7 * c + 9 * d)
            theta = np.where(act, theta - fix, theta)
            conv |= act & (np.abs(fix) < 1e-8)
        scale = np.where(newton, tan(theta) / td, 0.0)
        flipped = ((td < 0) & (theta > 0)) | ((td > 0) & (theta < 0))
        ok = conv & ~flipped
        if info is not None:
            info["unconverged"], info["flipped"] = ~conv, flipped
        pux, puy = pwx * scale, pwy * scale
        prx = _mv(nfx, 0.0, ncx, pux, puy)
        pry = _mv(0.0, nfy, ncy, pux, puy)
        prz = _mv(0.0, 0.0, 1.0, pux, puy)
        fx_, fy_ = prx / prz, pry / prz
        return np.stack([np.where(ok, fx_, FAIL), np.where(ok, fy_, FAIL)], axis=1).astype(np.float32)


def undistort_points(pts, K, model, k, p=(0.0, 0.0), new_K=None, tan=np.tan, info=None):
    """the model's output for float32 points [n, 2]; K, new_K 3x3 (new_K None or all zero: K); k: k1..k6 (radtan) or k1..k4 (fisheye)"""
    K = np.asarray(K, np.float64).reshape(3, 3)
    nK = K if new_K is None or not np.any(new_K) else np.asarray(new_K, np.float64).reshape(3, 3)
    P = (nK[0, 0], nK[1, 1], nK[0, 2], nK[1, 2])
    pts = np.asarray(pts, np.float32).reshape(-1, 2)
    k = [float(v) for v in k] + [0.0] * 6
    if model == FISHEYE:
        return fisheye(pts, K[0, 0], K[1, 1], K[0, 2], K[1, 2], k[:4], P, tan, info)
    return radtan(pts, K[0, 0], K[1, 1], K[0, 2], K[1, 2], k[:6], p, P, info)


def cv2_undistort_points(cv2, pts, K, model, k, p=(0.0, 0.0), new_K=None):
    """what OpenCV returns for the same inputs (float32 points, double K / D / P)"""
    K = np.asarray(K, np.float64).reshape(3, 3)
    P = K if new_K is None or not np.any(new_K) else np.asarray(new_K, np.float64).reshape(3, 3)
    src = np.ascontiguousarray(np.asarray(pts, np.float32).reshape(-1, 1, 2))
    k = [float(v) for v in k] + [0.0] * 6
    if model == FISHEYE:
        out = cv2.fisheye.undistortPoints(src, K, np.array(k[:4], np.float64), R=np.eye(3), P=P)
    else:
        D = np.array([k[0], k[1], p[0], p[1], k[2]] + ([k[3], k[4], k[5]] if any(k[3:6]) else []), np.float64)
        out = cv2.undistortPoints(src, K, D, None, P)
    return np.asarray(out, np.float32).reshape(-1, 2)


def same(a, b):
    """bit-identical float32 arrays, every NaN equal to every NaN"""
    a = np.asarray(a, np.float32)
    b = np.asarray(b, np.float32)
    na, nb = np.isnan(a), np.isnan(b)
    return a.shape == b.shape and np.array_equal(na, nb) and np.array_equal(a.view(np.uint32)[~na], b.view(np.uint32)[~nb])
