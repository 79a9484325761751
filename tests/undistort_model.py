"""numpy restatement of the lens undistortion (line3dpp_b200/csrc/l3d_undistort.cu: ud_map_point / ud_fix / ud_entry / ud_tap_sum;
DESIGN.md §4a).  TEST INFRASTRUCTURE: the map formula OpenCV's initUndistortRectifyMap evaluates for fixed-point (CV_16SC2 + CV_16UC1)
maps, written out in double precision without fused multiply-adds, and cv::remap's INTER_LINEAR / BORDER_CONSTANT tap sum for 8-bit
images.  Also the integer test images, so that every machine rebuilds the same pixels."""
import hashlib

import numpy as np

INT_MIN = -2 ** 31


def make_image(h, w, c, seed=0):
    """uint8 [h, w] or [h, w, 3]: an integer hash of (x, y, channel, seed), no random-number stream"""
    y, x, ch = np.meshgrid(np.arange(h, dtype=np.uint64), np.arange(w, dtype=np.uint64), np.arange(c, dtype=np.uint64), indexing="ij")
    m = np.uint64(0xFFFFFFFF)
    v = (x * np.uint64(73856093)) ^ (y * np.uint64(19349663)) ^ ((ch + np.uint64(seed) * np.uint64(7)) * np.uint64(83492791))
    v &= m
    v = ((v ^ (v >> np.uint64(13))) * np.uint64(0x5BD1E995)) & m
    v ^= v >> np.uint64(15)
    img = (v & np.uint64(255)).astype(np.uint8)
    return img[:, :, 0] if c == 1 else img


def inverse_k(fx, fy, cx, cy):
    """ir0, ir2, ir4, ir5 of inv([[fx,0,cx],[0,fy,cy],[0,0,1]]) by cofactors over the determinant (OpenCV's 3x3 inversion)"""
    d = 1.0 / (fx * fy)
    return fy * d, -(cx * fy) * d, fx * d, -(fx * cy) * d


def fix32(t):
    """cvRound(t * 32): round half to even; not finite or outside int32 -> INT_MIN"""
    r = np.rint(t * 32.0)
    ok = (r >= -2147483648.0) & (r <= 2147483647.0)
    return np.where(ok, r, float(INT_MIN)).astype(np.int64)


def fixed_point_uv(w, h, fx, fy, cx, cy, k1, k2, k3, p1, p2):
    """(iu, iv) int64 [h, w]: the source position of every destination pixel in 1/32 px, every term evaluated"""
    ir0, ir2, ir4, ir5 = inverse_k(fx, fy, cx, cy)
    with np.errstate(over="ignore", invalid="ignore"):
        x = (np.arange(w, dtype=np.float64) * ir0 + ir2)[None, :]
        y = (np.arange(h, dtype=np.float64) * ir4 + ir5)[:, None]
        x2, y2 = x * x, y * y
        r2 = x2 + y2
        _2xy = 2.0 * x * y
        kr = 1.0 + ((k3 * r2 + k2) * r2 + k1) * r2
        xd = x * kr + p1 * _2xy + p2 * (r2 + 2.0 * x2)
        yd = y * kr + p1 * (r2 + 2.0 * y2) + p2 * _2xy
        return fix32(fx * xd + cx), fix32(fy * yd + cy)


def maps_from_uv(iu, iv):
    """OpenCV's fixed-point maps: map_xy int16 [h, w, 2] (saturated), map_frac uint16 [h, w] = (iv & 31) * 32 + (iu & 31)"""
    xy = np.stack([np.clip(iu >> 5, -32768, 32767), np.clip(iv >> 5, -32768, 32767)], axis=-1).astype(np.int16)
    return xy, ((iv & 31) * 32 + (iu & 31)).astype(np.uint16)


def undistort_maps(w, h, fx, fy, cx, cy, k1=0.0, k2=0.0, k3=0.0, p1=0.0, p2=0.0):
    return maps_from_uv(*fixed_point_uv(w, h, fx, fy, cx, cy, k1, k2, k3, p1, p2))


def remap(src, map_xy, map_frac):
    """cv::remap(src, map_xy, map_frac, INTER_LINEAR, BORDER_CONSTANT, 0) for uint8 [h, w] or [h, w, 3]"""
    img = src if src.ndim == 3 else src[:, :, None]
    H, W = img.shape[:2]
    X, Y = map_xy[..., 0].astype(np.int64), map_xy[..., 1].astype(np.int64)
    tx, ty = (map_frac & 31).astype(np.int64), (map_frac >> 5).astype(np.int64)
    acc = np.zeros(map_frac.shape + (img.shape[2],), np.int64)
    for dx, dy, wgt in ((0, 0, (32 - tx) * (32 - ty) * 32), (1, 0, tx * (32 - ty) * 32), (0, 1, (32 - tx) * ty * 32), (1, 1, tx * ty * 32)):
        xx, yy = X + dx, Y + dy
        inside = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
        tap = img[np.where(inside, yy, 0), np.where(inside, xx, 0)].astype(np.int64)
        acc += (wgt * inside)[..., None] * tap
    out = np.clip((acc + 16384) >> 15, 0, 255).astype(np.uint8)
    return out if src.ndim == 3 else out[:, :, 0]


def apply_corrections(map_xy, map_frac, idx, xy, frac):
    """the model's maps with the entries of another build (flat pixel index idx) put in"""
    a, b = map_xy.reshape(-1, 2).copy(), map_frac.reshape(-1).copy()
    a[idx], b[idx] = xy, frac
    return a.reshape(map_xy.shape), b.reshape(map_frac.shape)


def sha(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def case_params(g, name):
    """(w, h, c, K 3x3, radial[3], tangential[2]) of one case of tests/golden/ref_undistort_v1.npz"""
    p = g[f"{name}/size"]
    return int(p[0]), int(p[1]), int(p[2]), g[f"{name}/K"], g[f"{name}/radial"], g[f"{name}/tangential"]


def model_maps_for(w, h, K, radial, tangential):
    return undistort_maps(w, h, float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), float(radial[0]), float(radial[1]), float(radial[2]),
                          float(tangential[0]), float(tangential[1]))
