"""float64 numpy model of l3d_pose_neighbors (DESIGN.md §6d) in the library's operation order, and scene builders for its tests.

Steps 1-3 (samples, back-projection, observation) are IEEE double adds, multiplies and divides in the order of csrc/l3d_pose.cu, so
every observation is reproduced bit for bit.  Steps 4-5 restate find_visual_neighbors of csrc/line3d_host.cc: the camera quantities of
addImage (R^T K^-1 with the adjugate inverse, C = R^T (-t)), the float score, acos of the axes, the 0.8 cut, the distance resort and
the greedy baseline loop.  `reference_neighbors` is a second, loop-and-set restatement of findVisualNeighborsFromWPs (line3D.cc:578-699)
fed the virtual world points, for the CPU tests to set against `select`."""
from __future__ import annotations

import math

import numpy as np

f32 = np.float32


class Views:
    """n posed views: cam_ids (n,) uint32, K (n,3,3), R (n,3,3), t (n,3), width / height (n,) int, depth (n,) float64"""

    def __init__(self, cam_ids, K, R, t, width, height, depth):
        n = len(cam_ids)
        self.cam_ids = np.asarray(cam_ids, np.uint32)
        self.K = np.asarray(K, np.float64).reshape(n, 3, 3)
        self.R = np.asarray(R, np.float64).reshape(n, 3, 3)
        self.t = np.asarray(t, np.float64).reshape(n, 3)
        self.width = np.broadcast_to(np.asarray(width, np.int64), (n,)).copy()
        self.height = np.broadcast_to(np.asarray(height, np.int64), (n,)).copy()
        self.depth = np.broadcast_to(np.asarray(depth, np.float64), (n,)).copy()

    def __len__(self):
        return len(self.cam_ids)

    def subset(self, idx):
        idx = list(idx)
        return Views(self.cam_ids[idx], self.K[idx], self.R[idx], self.t[idx], self.width[idx], self.height[idx], self.depth[idx])


# ---- steps 1-3 ---------------------------------------------------------------------------------------------------------------------
def sample_points(V: Views, gx: int, gy: int) -> np.ndarray:
    """(n * gx * gy, 3) virtual points; point i * G + s is view i's sample s = r * gx + c"""
    G = gx * gy
    s = np.arange(G)
    c, r = (s % gx).astype(np.float64), (s // gx).astype(np.float64)
    out = np.empty((len(V) * G, 3))
    for i in range(len(V)):
        K, R, t = V.K[i], V.R[i], V.t[i]
        fx, fy, cx, cy, sk = K[0, 0], K[1, 1], K[0, 2], K[1, 2], K[0, 1]
        u = (c + 0.5) * float(V.width[i]) / float(gx)
        v = (r + 0.5) * float(V.height[i]) / float(gy)
        yn = (v - cy) / fy
        xn = ((u - cx) - sk * yn) / fx
        z = V.depth[i]
        d0, d1, d2 = z * xn - t[0], z * yn - t[1], np.full(G, z - t[2])
        for k in range(3):
            out[i * G:(i + 1) * G, k] = (R[0, k] * d0 + R[1, k] * d1) + R[2, k] * d2
    return out


def sees(V: Views, j: int, X: np.ndarray) -> np.ndarray:
    """bool per point: view j sees X (depth > 0, inside [0, width) x [0, height)); its own points are not special here"""
    K, R, t = V.K[j], V.R[j], V.t[j]
    x, y, z = X[:, 0], X[:, 1], X[:, 2]
    c2 = ((R[2, 0] * x + R[2, 1] * y) + R[2, 2] * z) + t[2]
    c0 = ((R[0, 0] * x + R[0, 1] * y) + R[0, 2] * z) + t[0]
    c1 = ((R[1, 0] * x + R[1, 1] * y) + R[1, 2] * z) + t[1]
    with np.errstate(divide="ignore", invalid="ignore"):
        u = ((K[0, 0] * c0 + K[0, 1] * c1) + K[0, 2] * c2) / c2
        v = (K[1, 1] * c1 + K[1, 2] * c2) / c2
    return (c2 > 0) & (u >= 0) & (u < float(V.width[j])) & (v >= 0) & (v < float(V.height[j]))


def observations(V: Views, gx: int, gy: int, views=None, X=None) -> np.ndarray:
    """bool (P, len(views)): point p observed by view views[k] (its own view always); views None: all"""
    G = gx * gy
    X = sample_points(V, gx, gy) if X is None else X
    views = range(len(V)) if views is None else views
    own = np.arange(len(X)) // G
    return np.stack([sees(V, j, X) | (own == j) for j in views], axis=1)


def counts(V: Views, gx: int, gy: int, views=None):
    """(n_i (n,) of every view, the rows of common (len(views), n) of `views` (default all), zero at (i, i))"""
    O = observations(V, gx, gy).astype(np.float64)          # exact: counts stay far below 2^53
    n = O.sum(axis=0).astype(np.int64)
    views = list(range(len(V))) if views is None else list(views)
    cm = np.rint(O[:, views].T @ O).astype(np.int64)
    cm[np.arange(len(views)), views] = 0
    return n, cm


# ---- camera quantities of addImage (csrc/line3d_host.cc), scalar doubles in its order ------------------------------------------------
def _matmul(a, b):
    r = [[0.0] * 3 for _ in range(3)]
    for i in range(3):
        for j in range(3):
            s = 0.0
            for k in range(3):
                s += a[i][k] * b[k][j]
            r[i][j] = s
    return r


def _matvec(a, v):
    return [a[0][0] * v[0] + a[0][1] * v[1] + a[0][2] * v[2], a[1][0] * v[0] + a[1][1] * v[1] + a[1][2] * v[2],
            a[2][0] * v[0] + a[2][1] * v[1] + a[2][2] * v[2]]


def _inverted(a):
    c00 = a[1][1] * a[2][2] - a[1][2] * a[2][1]
    c01 = a[1][2] * a[2][0] - a[1][0] * a[2][2]
    c02 = a[1][0] * a[2][1] - a[1][1] * a[2][0]
    i = 1.0 / (a[0][0] * c00 + a[0][1] * c01 + a[0][2] * c02)
    r = [[0.0] * 3 for _ in range(3)]
    r[0][0], r[1][0], r[2][0] = c00 * i, c01 * i, c02 * i
    r[0][1] = (a[0][2] * a[2][1] - a[0][1] * a[2][2]) * i
    r[1][1] = (a[0][0] * a[2][2] - a[0][2] * a[2][0]) * i
    r[2][1] = (a[0][1] * a[2][0] - a[0][0] * a[2][1]) * i
    r[0][2] = (a[0][1] * a[1][2] - a[0][2] * a[1][1]) * i
    r[1][2] = (a[0][2] * a[1][0] - a[0][0] * a[1][2]) * i
    r[2][2] = (a[0][0] * a[1][1] - a[0][1] * a[1][0]) * i
    return r


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _unit(a):
    n2 = _dot(a, a)
    if n2 > 0:
        n = math.sqrt(n2)
        return [a[0] / n, a[1] / n, a[2] / n]
    return a


class Cam:
    """what find_visual_neighbors reads of a view: R, t, C, the optical axis ray"""

    def __init__(self, K, R, t):
        K = [[float(K[0, 0]), float(K[0, 1]), float(K[0, 2])], [0.0, float(K[1, 1]), float(K[1, 2])], [0.0, 0.0, 1.0]]
        self.R = [[float(x) for x in row] for row in R]
        self.t = [float(x) for x in t]
        Rt = [[self.R[j][i] for j in range(3)] for i in range(3)]
        RtKinv = _matmul(Rt, _inverted(K))
        self.C = _matvec(Rt, [self.t[0] * -1.0, self.t[1] * -1.0, self.t[2] * -1.0])
        self.axis = _unit(_matvec(RtKinv, [K[0][2], K[1][2], 1.0]))


def cams_of(V: Views):
    return [Cam(V.K[i], V.R[i], V.t[i]) for i in range(len(V))]


def axis_angle(a: Cam, b: Cam):
    return f32(math.acos(min(max(_dot(a.axis, b.axis), -1.0), 1.0)))


def dist_score(a: Cam, b: Cam):
    ct = _matvec(a.R, b.C)
    ct = [ct[k] + a.t[k] for k in range(3)]
    return f32(abs(f32(ct[0])) + abs(f32(ct[1])))


def baseline(a: Cam, b: Cam):
    d = [a.C[k] - b.C[k] for k in range(3)]
    return f32(math.sqrt(_dot(d, d)))


def score(common, ni, nj):
    return f32(2.0) * f32(common) / f32(ni + nj)


# ---- step 5 ------------------------------------------------------------------------------------------------------------------------
def select_one(i, cams, cam_ids, n, common_row, num_neighbors):
    """find_visual_neighbors of view i given its row of common counts: the sorted camIDs of its neighbours"""
    ranked = [(int(cam_ids[j]), score(int(common_row[j]), int(n[i]), int(n[j])), j) for j in np.argsort(cam_ids, kind="stable")
              if j != i and common_row[j] > 4]
    ranked.sort(key=lambda c: -c[1])                                     # stable: ties stay in ascending camID
    cand = [(cam, s, axis_angle(cams[i], cams[j]), dist_score(cams[i], cams[j]), j) for cam, s, j in ranked]
    cand = [c for c in cand if c[2] < f32(1.571)]
    if len(cand) > num_neighbors:
        all_ = list(cand)
        t = f32(0.8) * cand[0][1]
        nbig = 0
        while nbig < len(cand) and cand[nbig][1] > t:
            nbig += 1
        cand = sorted(cand[:nbig], key=lambda c: -c[3])
        cand = cand[:num_neighbors // 2] + all_
    out, used = set(), []
    for cam, _, _, _, j in cand:
        if len(out) >= num_neighbors:
            break
        if cam in out or not baseline(cams[i], cams[j]) > f32(0.1):
            continue
        if all(baseline(cams[i], cams[u]) > f32(0.1) for u in used):
            out.add(cam)
            used.append(j)
    return sorted(out)


def select(V: Views, n, common, num_neighbors, views=None):
    """neighbour lists (sorted camIDs) of `views` (default all); n: n_i of every view; common: the rows of those views"""
    cams = cams_of(V)
    views = range(len(V)) if views is None else views
    return [select_one(i, cams, V.cam_ids, n, common[k], num_neighbors) for k, i in enumerate(views)]


def pose_neighbors(V: Views, gx, gy, num_neighbors):
    n, cm = counts(V, gx, gy)
    return select(V, n, cm, num_neighbors)


# ---- the virtual world points as a frontend would pass them, and the reference's loop ----------------------------------------------
def world_point_lists(V: Views, gx, gy):
    """per view the IDs (i * G + s) of the virtual points it observes, ascending"""
    O = observations(V, gx, gy)
    return [np.flatnonzero(O[:, j]).astype(np.uint32) for j in range(len(V))]


def reference_neighbors(V: Views, wps, num_neighbors):
    """findVisualNeighborsFromWPs (line3D.cc:578-699) statement by statement over views2worldpoints_ = wps (by view index, camIDs
    from V), worldpoints2views_ built as addImage builds it, num_worldpoints_ = the list sizes"""
    cams = cams_of(V)
    by_cam = {int(V.cam_ids[i]): i for i in range(len(V))}
    wp2views = {}
    for cam in sorted(by_cam):
        for wp in wps[by_cam[cam]]:
            wp2views.setdefault(int(wp), []).append(cam)
    out = []
    for i in range(len(V)):
        camID = int(V.cam_ids[i])
        commonWPs = {}
        for wpID in wps[i]:
            for vID in wp2views[int(wpID)]:
                if vID != camID:
                    commonWPs[vID] = commonWPs.get(vID, 0) + 1
        if len(commonWPs) == 0:
            out.append([])
            continue
        used_neighbors = set()
        neighbors = []
        for vID in sorted(commonWPs):
            num_common_wps = commonWPs[vID]
            j = by_cam[vID]
            vn = dict(camID=vID, score=f32(2.0) * f32(num_common_wps) / f32(len(wps[i]) + len(wps[j])),
                      axisAngle=axis_angle(cams[i], cams[j]), distance_score=dist_score(cams[i], cams[j]))
            if vn["axisAngle"] < f32(1.571) and num_common_wps > 4:
                neighbors.append(vn)
        neighbors = sorted(neighbors, key=lambda a: -a["score"])
        if len(neighbors) > num_neighbors:
            neighbors_tmp = list(neighbors)
            score_t = f32(0.80) * neighbors[0]["score"]
            num_bigger_t = 0
            while num_bigger_t < len(neighbors) and neighbors[num_bigger_t]["score"] > score_t:
                num_bigger_t += 1
            neighbors = neighbors[:num_bigger_t]
            neighbors = sorted(neighbors, key=lambda a: -a["distance_score"])
            if len(neighbors) > num_neighbors // 2:
                neighbors = neighbors[:num_neighbors // 2]
            neighbors = neighbors + neighbors_tmp
        min_baseline = f32(0.1)
        k = 0
        while k < len(neighbors) and len(used_neighbors) < num_neighbors:
            vn = neighbors[k]
            if vn["camID"] not in used_neighbors and baseline(cams[i], cams[by_cam[vn["camID"]]]) > min_baseline:
                valid = True
                for u in sorted(used_neighbors):
                    if not valid:
                        break
                    if not baseline(cams[i], cams[by_cam[u]]) > min_baseline:
                        valid = False
                if valid:
                    used_neighbors.add(vn["camID"])
            k += 1
        out.append(sorted(used_neighbors))
    return out


# ---- scenes ------------------------------------------------------------------------------------------------------------------------
def look_at(C, target=(0.0, 0.0, 0.0), up=(0.0, 1.0, 0.0)):
    C = np.asarray(C, np.float64)
    z = np.asarray(target, np.float64) - C
    z /= np.linalg.norm(z)
    x = np.cross(np.asarray(up, np.float64), z)
    x /= np.linalg.norm(x)
    y = np.cross(z, x)
    R = np.stack([x, y, z])
    return R, -R @ C


def intrinsics(f, w, h, skew=0.0):
    return np.array([[f, skew, w / 2.0], [0.0, f, h / 2.0], [0.0, 0.0, 1.0]])


def ring(V, radius=4.0, w=640, h=480, f=500.0, depth=4.0, seed=0, cam_ids=None, jitter=0.2):
    """V views on a circle looking at the centre, heights jittered"""
    rng = np.random.default_rng(seed)
    Rs, ts = [], []
    for i in range(V):
        th = 2.0 * np.pi * i / V
        R, t = look_at([radius * np.cos(th), rng.uniform(-jitter, jitter), radius * np.sin(th)])
        Rs.append(R); ts.append(t)
    ids = np.arange(V) if cam_ids is None else cam_ids
    return Views(ids, np.repeat(intrinsics(f, w, h)[None], V, 0), Rs, ts, w, h, depth)


def grid_survey(nx, ny, spacing=1.0, height=10.0, w=800, h=600, f=600.0, seed=0):
    """nadir views on an nx x ny grid at `height` over the plane z = 0 (a drone survey with parallel strips)"""
    rng = np.random.default_rng(seed)
    Rs, ts = [], []
    R = np.array([[1.0, 0, 0], [0, -1.0, 0], [0, 0, -1.0]])      # looking down -z
    for a in range(ny):
        for b in range(nx):
            C = np.array([b * spacing, a * spacing, height]) + rng.normal(scale=0.02, size=3)
            Rs.append(R); ts.append(-R @ C)
    V = nx * ny
    return Views(np.arange(V), np.repeat(intrinsics(f, w, h)[None], V, 0), Rs, ts, w, h, height)


def random_poses(V, w=320, h=240, seed=0, spread=3.0):
    """cameras around the origin, each looking at a random point near it, random focal, skew, sizes and depths"""
    rng = np.random.default_rng(seed)
    Ks, Rs, ts, ws, hs, ds = [], [], [], [], [], []
    for _ in range(V):
        C = rng.normal(size=3) * spread
        R, t = look_at(C, rng.normal(size=3) * 0.5)
        ww, hh = int(rng.integers(w // 2, w * 2)), int(rng.integers(h // 2, h * 2))
        Ks.append(np.array([[rng.uniform(200, 600), rng.uniform(-2, 2), rng.uniform(0.3, 0.7) * ww],
                            [0, rng.uniform(200, 600), rng.uniform(0.3, 0.7) * hh], [0, 0, 1.0]]))
        Rs.append(R); ts.append(t); ws.append(ww); hs.append(hh); ds.append(np.linalg.norm(C) * rng.uniform(0.5, 1.5))
    return Views(rng.permutation(10 * V)[:V], Ks, Rs, ts, ws, hs, ds)
