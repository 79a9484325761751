"""An independent extended-precision model of tie-point triangulation and per-camera median depths (l3d_triangulate_points,
l3d_median_depths, DESIGN.md §6b), and problem builders, each named by the kernel path it reaches.

The model forms A^T A of linearHomTriangulation (main_pix4d.cpp:34-70: per observation the rows Sx P[cam], Sx = [[0,-1,y],[1,0,-x]])
exactly from the double inputs, in integers, and takes its eigen-decomposition with mpmath at PREC bits.  It shares no arithmetic with
the device's Jacobi.  mpmath costs about 5 ms a point, so it runs on a stratified subset (every constructed ill-conditioned or
degenerate point, the points numpy finds worst conditioned, a random sample of the rest); numpy's eigh of the double A^T A stands in
for the bulk, which is well conditioned.

The contract the tests hold the device to: ||X - X*|| <= C 2^-52 kappa sqrt(1 + ||X*||^2) (1 + ||X*||) with kappa = lambda_max /
(lambda_2 - lambda_1) of the exact A^T A.  An eigenvector of a matrix perturbed by eps ||A^T A|| moves by about eps kappa, and X = v.xyz /
v.w turns that into the bound above (|v.w| = 1 / sqrt(1 + ||X||^2)).  The bound grows like ||X*||^2: for distant points it allows
more than ||X*|| itself, so there the tests hold the direction of X to its own bound (Model.direction_ratio).
"""
from __future__ import annotations

import os

import mpmath
import numpy as np

EPS = 2.0 ** -52
L3D_EPS = 1e-12                 # the reference's validity threshold on |X| (commons.h:95)
PREC = 256

# cub::DeviceSegmentedSort for 4-byte keys and no values under Policy860, the policy of sm_86 and later
# (cub/device/dispatch/tuning/tuning_segmented_sort.cuh; tests/test_tri_model_cpu.py reads the header and checks these)
CUB_PARTITIONING_THRESHOLD = 500      # more segments than this: partitioned into small, medium and large segments
CUB_SMALL_MAX = 2 * 9                 # a small segment: a sub-warp of 2 threads x 9 items
CUB_MEDIUM_MAX = 16 * 7               # a medium segment: 16 threads x 7 items; also the single-warp limit of the unpartitioned kernel
CUB_LARGE_TILE = 256 * 23             # a segment shorter than this is sorted in one block-radix tile, one this long or longer in several passes
CUB_TUNING_HEADER = "/usr/local/cuda/include/cub/device/dispatch/tuning/tuning_segmented_sort.cuh"


# ---------------------------------------------------------------------------------------------- exact normal matrices
def _exact_ints(a):
    """a (finite float64) as integers N and one shift s with a == N * 2^-s exactly"""
    ratios = [float(v).as_integer_ratio() for v in np.asarray(a, np.float64).ravel()]
    s = max((d.bit_length() - 1 for _, d in ratios), default=0)
    return np.array([n << (s - (d.bit_length() - 1)) for n, d in ratios], dtype=object).reshape(np.shape(a)), s


def normal_matrix_exact(cams, xy, P):
    """A^T A of one point exactly: (N, s) with A^T A == N * 2^-s, N a 4x4 object array of Python integers"""
    M, sp = _exact_ints(P[np.asarray(cams)].reshape(-1, 12))
    Y, sx = _exact_ints(np.asarray(xy, np.float64).reshape(-1, 2))
    x, y = Y[:, 0:1], Y[:, 1:2]
    r1 = -M[:, 4:8] * (1 << sx) + y * M[:, 8:12]          # rows scaled by 2^(sp + sx)
    r2 = M[:, 0:4] * (1 << sx) - x * M[:, 8:12]
    return r1.T.dot(r1) + r2.T.dot(r2), 2 * (sp + sx)


def _mp_matrix(N, s):
    return mpmath.matrix([[mpmath.ldexp(mpmath.mpf(int(N[r, c])), -s) for c in range(4)] for r in range(4)])


def point_exact(cams, xy, P):
    """the model of one point with at least three finite observations: X* (float64, +-inf where v.w == 0), the eigenvalues of A^T A
    in ascending order, |v.w| and kappa = lambda_max / (lambda_2 - lambda_1), all rounded from PREC bits"""
    with mpmath.workprec(PREC):
        A = _mp_matrix(*normal_matrix_exact(cams, xy, P))
        E, Q = mpmath.eigsy(A)
        order = sorted(range(4), key=lambda i: E[i])
        lam = [E[i] for i in order]
        v = [Q[r, order[0]] for r in range(4)]
        X = [float(v[k] / v[3]) if v[3] != 0 else (np.inf if v[k] > 0 else -np.inf if v[k] < 0 else np.nan) for k in range(3)]
        gap = lam[1] - lam[0]
        kappa = float(lam[3] / gap) if gap > 0 else np.inf
        return np.array(X), np.array([float(e) for e in lam]), float(abs(v[3])), kappa


def residual_ratio(cams, xy, P, X):
    """||A^T A v|| / ||A^T A|| (spectral norm) for v = (X, 1) / ||(X, 1)||: how far X is from the null space, for points whose null
    space has more than one dimension"""
    with mpmath.workprec(PREC):
        A = _mp_matrix(*normal_matrix_exact(cams, xy, P))
        v = mpmath.matrix([mpmath.mpf(float(X[0])), mpmath.mpf(float(X[1])), mpmath.mpf(float(X[2])), mpmath.mpf(1)])
        v = v / mpmath.norm(v)
        lmax = max(mpmath.eigsy(A, eigvals_only=True))
        return float(mpmath.norm(A * v) / lmax) if lmax > 0 else 0.0


# ---------------------------------------------------------------------------------------------- the model of a whole problem
def _numpy_model(ptr, cam, xy, P):
    """A^T A in double, eigh: X, kappa for every point (the bulk model)"""
    Pc = P.reshape(-1, 3, 4)[cam]
    r1 = -Pc[:, 1] + xy[:, 1:2] * Pc[:, 2]
    r2 = Pc[:, 0] - xy[:, 0:1] * Pc[:, 2]
    outer = np.einsum("ni,nj->nij", r1, r1) + np.einsum("ni,nj->nij", r2, r2)
    seg = np.repeat(np.arange(len(ptr) - 1), np.diff(ptr))
    A = np.zeros((len(ptr) - 1, 4, 4))
    np.add.at(A, seg, outer)
    A = np.where(np.isfinite(A).all(axis=(1, 2))[:, None, None], A, 0.0)
    w, V = np.linalg.eigh(A)
    v = V[:, :, 0]
    with np.errstate(divide="ignore", invalid="ignore"):
        return v[:, :3] / v[:, 3:], w[:, 3] / (w[:, 1] - w[:, 0])


class Model:
    """the model of every point of a problem: X (float64 [n, 3]), kappa, valid, and which points it holds to the bound (`bounded`),
    which to a residual (`null2`: a null space of two or more dimensions) and which to the rule for non-finite input (`nonfinite`).
    `exact` marks the points mpmath solved."""

    def __init__(self, ptr, cam, xy, P, special=(), null2=(), n_sample=200, n_worst=200, seed=0):
        ptr, cam = np.asarray(ptr, np.int64), np.asarray(cam, np.int32)
        xy, P = np.asarray(xy, np.float64).reshape(-1, 2), np.asarray(P, np.float64).reshape(-1, 12)
        n = len(ptr) - 1
        cnt = np.diff(ptr)
        known = np.ones(n, bool)
        bad_cam = (cam < 0) | (cam >= len(P))
        finite_obs = np.isfinite(xy).all(1) & ~bad_cam
        finite_obs[~bad_cam] &= np.isfinite(P[cam[~bad_cam]]).all(1)
        seg = np.repeat(np.arange(n), cnt)
        np.logical_and.at(known, seg, ~bad_cam)
        finite = np.ones(n, bool)
        np.logical_and.at(finite, seg, finite_obs)
        self.ptr, self.cam, self.xy, self.P = ptr, cam, xy, P
        self.enough = (cnt >= 3) & known
        self.nonfinite = self.enough & ~finite
        self.null2 = np.zeros(n, bool)
        self.null2[list(null2)] = True
        ok = self.enough & finite
        camc = np.where(bad_cam, 0, cam)
        self.X, self.kappa = _numpy_model(ptr, camc, np.where(finite_obs[:, None], xy, 0.0), np.where(np.isfinite(P), P, 0.0))
        self.X[~ok] = 0.0
        self.kappa[~ok] = np.nan
        self.vw = np.full(n, np.nan)
        self.exact = np.zeros(n, bool)
        rng = np.random.default_rng(seed)
        cand = np.flatnonzero(ok & ~self.null2)
        pick = set(int(i) for i in special if ok[i] and not self.null2[i])
        if len(cand):
            pick |= set(int(i) for i in rng.choice(cand, min(n_sample, len(cand)), replace=False))
            kap = np.nan_to_num(self.kappa[cand], nan=np.inf)
            pick |= set(int(i) for i in cand[np.argsort(-kap)[:n_worst]])
        for i in sorted(pick):
            b, e = ptr[i], ptr[i + 1]
            X, _, vw, kappa = point_exact(cam[b:e], xy[b:e], P)
            self.X[i], self.vw[i], self.kappa[i], self.exact[i] = X, vw, kappa, True
        self.bounded = ok & ~self.null2
        nrm = np.sqrt((self.X * self.X).sum(1))
        self.valid = (ok & (nrm > L3D_EPS)).astype(np.int32)

    def bound(self, C):
        """C 2^-52 kappa sqrt(1 + ||X*||^2) (1 + ||X*||) for every bounded point (inf where X* is infinite)"""
        nrm = np.sqrt((self.X * self.X).sum(1))
        with np.errstate(invalid="ignore", over="ignore"):
            return C * EPS * self.kappa * np.sqrt(1.0 + nrm * nrm) * (1.0 + nrm)

    def ratio(self, X):
        """||X - X*|| / (2^-52 kappa sqrt(1 + ||X*||^2) (1 + ||X*||)) on the bounded points whose X* is finite (nan elsewhere)"""
        with np.errstate(invalid="ignore", over="ignore"):
            r = np.sqrt(((np.asarray(X) - self.X) ** 2).sum(1)) / self.bound(1.0)
        r[~self.bounded | ~np.isfinite(self.X).all(1)] = np.nan
        return r

    def direction_ratio(self, X):
        """||X / ||X|| - X* / ||X*|| || / (2^-52 kappa 2 sqrt(1 + ||X*||^2) / ||X*||) on the bounded points where X and X* are finite and
        nonzero (nan elsewhere): the direction of v.xyz moves by at most 2 ||dv|| / ||v.xyz||, so this stays meaningful for distant
        points, where the bound on the position allows more than ||X*|| itself"""
        X = np.asarray(X, np.float64)
        with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
            nx, ns = np.linalg.norm(X, axis=1), np.linalg.norm(self.X, axis=1)
            d = np.linalg.norm(X / nx[:, None] - self.X / ns[:, None], axis=1)
            r = d / (EPS * self.kappa * 2.0 * np.sqrt(1.0 + ns * ns) / ns)
        r[~self.bounded | ~np.isfinite(X).all(1) | ~np.isfinite(self.X).all(1) | (nx == 0) | (ns == 0)] = np.nan
        return r

    def flag_decidable(self, C):
        """the bounded points whose ||X*|| is not within the bound of L3D_EPS, so that their valid flag is determined"""
        nrm = np.sqrt((self.X * self.X).sum(1))
        with np.errstate(invalid="ignore"):
            return self.bounded & (np.abs(nrm - L3D_EPS) > self.bound(C))


# ---------------------------------------------------------------------------------------------- median depths
def median_model(lptr, lpts, X, valid, Cs):
    """main_pix4d.cpp:386-418: per camera the float depths (float)|X - C| (a float64 norm, summed x, y, z) of the valid points of its
    list (an id outside [0, n) is not valid), sorted; (count, element [count / 2] or 0)"""
    X, Cs = np.asarray(X, np.float64).reshape(-1, 3), np.asarray(Cs, np.float64).reshape(-1, 3)
    n, nc = len(X), len(lptr) - 1
    cnt, med = np.zeros(nc, np.int32), np.zeros(nc, np.float32)
    for c in range(nc):
        ids = np.asarray(lpts[lptr[c]:lptr[c + 1]], np.int64)
        ids = ids[(ids >= 0) & (ids < n)]
        ids = ids[np.asarray(valid)[ids] != 0]
        d = X[ids] - Cs[c]
        with np.errstate(over="ignore"):
            dep = np.sort(np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]).astype(np.float32))
        cnt[c] = len(dep)
        med[c] = dep[len(dep) // 2] if len(dep) else np.float32(0)
    return cnt, med


def cub_limits(path=CUB_TUNING_HEADER):
    """(partitioning threshold, small max, medium max, large tile) of Policy860 for 4-byte keys, read from the cub header"""
    import re
    txt = open(path).read()
    body = txt[txt.index("struct Policy860"):]
    body = body[:body.index("};")]
    num = lambda pat: int(re.search(pat, body, re.S).group(1))
    threshold = num(r"PARTITIONING_THRESHOLD\s*=\s*(\d+)")
    block = num(r"BLOCK_THREADS\s*=\s*(\d+)")
    items = num(r"AgentRadixSortDownsweepPolicy<\s*BLOCK_THREADS,\s*(\d+)")
    small_items = num(r"ITEMS_PER_SMALL_THREAD\s*=\s*Nominal4BItemsToItems<DominantT>\(LARGE_ITEMS \? \d+ : (\d+)\)")
    medium_items = num(r"ITEMS_PER_MEDIUM_THREAD\s*=\s*Nominal4BItemsToItems<DominantT>\(LARGE_ITEMS \? \d+ : (\d+)\)")
    small_threads = num(r"AgentSubWarpMergeSortPolicy<LARGE_ITEMS \? \d+ : (\d+)")
    medium_threads = num(r"// Medium policy\s*AgentSubWarpMergeSortPolicy<(\d+)")
    return threshold, small_threads * small_items, medium_threads * medium_items, block * items


def tr_smem_max():
    """TR_SMEM_MAX of csrc/l3d_triangulate.cu: the bytes of camera matrices k_triangulate stages in shared memory"""
    import re
    src = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "line3dpp_b200", "csrc", "l3d_triangulate.cu")
    a, b = re.search(r"#define TR_SMEM_MAX \((\d+) \* (\d+)\)", open(src).read()).groups()
    return int(a) * int(b)


def cub_header_present():
    return os.path.exists(CUB_TUNING_HEADER)


# ---------------------------------------------------------------------------------------------- problem builders
def look_at(C, target, up=(0.0, 0.0, 1.0)):
    """rows x, y, z of a camera rotation whose z axis points from C to target"""
    z = np.asarray(target, np.float64) - C
    z /= np.linalg.norm(z)
    x = np.cross(up, z)
    if np.linalg.norm(x) < 1e-9:
        x = np.cross((0.0, 1.0, 0.0), z)
    x /= np.linalg.norm(x)
    return np.stack([x, np.cross(z, x), z])


def projection(K, R, C):
    return K @ np.hstack([R, (-R @ C)[:, None]])


def project(P, Xh):
    h = P @ Xh
    return h[:2] / h[2]


class Problem:
    """a triangulation problem: CSR observations (ptr, cam, xy), camera matrices P [cams, 3, 4] and centres, and `tags`: the point
    indices of every constructed case, by name"""

    def __init__(self, obs, P, centres=None, tags=None):
        cnt = [len(o[0]) for o in obs]
        self.ptr = np.zeros(len(obs) + 1, np.int64)
        self.ptr[1:] = np.cumsum(cnt)
        self.cam = np.array([c for o in obs for c in o[0]], np.int32)
        self.xy = np.array([p for o in obs for p in o[1]], np.float64).reshape(-1, 2)
        self.P = np.asarray(P, np.float64).reshape(-1, 3, 4)
        self.centres = centres
        self.tags = tags or {}

    @property
    def n(self):
        return len(self.ptr) - 1

    def special(self):
        return sorted(set(i for v in self.tags.values() for i in v))


def pix4d_scale(n_points=4000, offset=(461234.5, 5254321.25, 412.0), seed=0, noise=0.3):
    """A georeferenced survey: 48 nadir cameras (f = 3600-4000 px) on a 6 x 8 grid 110 m above the ground and 24 oblique ones
    (f = 7800-8000 px, 45 degrees) on a ring, 4000 x 3000 images, ground points over 400 m x 300 m, every coordinate offset by
    `offset`.  Returns (world problem, the same problem with the offset subtracted, the points' true positions in the world)."""
    rng = np.random.default_rng(seed)
    off = np.asarray(offset, np.float64)
    cams = []
    for i in range(6):
        for j in range(8):
            C = np.array([-150 + 60.0 * i, -140 + 40.0 * j, 110 + rng.uniform(-2, 2)])
            R = look_at(C, C + np.array([rng.uniform(-4, 4), rng.uniform(-4, 4), -110]), up=(0.0, 1.0, 0.0))
            cams.append((rng.uniform(3600, 4000), R, C))
    for k in range(24):
        a = 2 * np.pi * k / 24
        C = np.array([260 * np.cos(a), 200 * np.sin(a), 150.0])
        cams.append((rng.uniform(7800, 8000), look_at(C, np.array([0.4 * C[0], 0.4 * C[1], 0.0])), C))
    Xs = np.stack([rng.uniform(-200, 200, n_points), rng.uniform(-150, 150, n_points), rng.uniform(-3, 8, n_points)], 1)
    Pw, Pl, Cw = [], [], []
    for f, R, C in cams:
        K = np.array([[f, 0, 2000 + rng.uniform(-20, 20)], [0, f, 1500 + rng.uniform(-20, 20)], [0, 0, 1]])
        Pw.append(projection(K, R, C + off)); Pl.append(projection(K, R, C)); Cw.append(C + off)
    Pl = np.stack(Pl)
    obs = []
    for X in Xs:
        h = Pl @ np.append(X, 1.0)
        xy = h[:, :2] / h[:, 2:]
        seen = np.flatnonzero((h[:, 2] > 0) & (xy[:, 0] >= 0) & (xy[:, 0] < 4000) & (xy[:, 1] >= 0) & (xy[:, 1] < 3000))
        seen = rng.permutation(seen)[:rng.integers(3, 25)]
        obs.append((seen.tolist(), (xy[seen] + rng.normal(0, noise, (len(seen), 2))).tolist()))
    world, local = Problem(obs, np.stack(Pw), np.stack(Cw)), Problem(obs, Pl, np.stack(Cw) - off)
    world.focal = local.focal = np.array([f for f, _, _ in cams])
    return world, local, Xs + off


def ill_conditioned(seed=1):
    """Points 50 m from three to five cameras whose baselines are 1e-1 down to 1e-7 of that depth (kappa about 1e2 to 1e14), with exact
    and with noisy (0.5 px) projections: tag 'ill'"""
    rng = np.random.default_rng(seed)
    K = np.array([[1200.0, 0, 960], [0, 1200.0, 540], [0, 0, 1]])
    P, obs = [], []
    for r in np.logspace(-1, -7, 25):
        for noisy in (False, True):
            X = rng.uniform(-5, 5, 3)
            d = rng.normal(size=3); d /= np.linalg.norm(d)
            ncam = int(rng.integers(3, 6))
            ids = []
            for _ in range(ncam):
                C = X - 50.0 * d + 50.0 * r * rng.uniform(-1, 1, 3)
                ids.append(len(P))
                P.append(projection(K, look_at(C, X + rng.uniform(-1, 1, 3)), C))
            xy = [project(P[c], np.append(X, 1.0)) + (rng.normal(0, 0.5, 2) if noisy else 0.0) for c in ids]
            obs.append((ids, xy))
    return Problem(obs, np.stack(P), tags={"ill": list(range(len(obs)))})


def near_infinity(seed=2):
    """Points 1e3 to 1e15 m away along a direction seen by four to six cameras 10 m apart, and exact points at infinity (w = 0): |v.w|
    from about 1e-3 down to 0: tags 'far' and 'infinite'"""
    rng = np.random.default_rng(seed)
    K = np.array([[1500.0, 0, 1000], [0, 1500.0, 750], [0, 0, 1]])
    Cs = [np.array([10.0 * np.cos(a), 10.0 * np.sin(a), 0.5 * np.sin(3 * a)]) for a in np.linspace(0, 2 * np.pi, 6, endpoint=False)]
    P = [projection(K, look_at(C, np.array([0.0, 0.0, 1e6])), C) for C in Cs]
    obs, far, inf = [], [], []
    for t in np.logspace(3, 15, 25):
        d = np.array([rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), 1.0]); d /= np.linalg.norm(d)
        ids = sorted(rng.choice(6, int(rng.integers(4, 7)), replace=False).tolist())
        far.append(len(obs))
        obs.append((ids, [project(P[c], np.append(t * d, 1.0)) + rng.normal(0, 0.2, 2) for c in ids]))
    for _ in range(6):
        d = np.array([rng.uniform(-0.3, 0.3), rng.uniform(-0.3, 0.3), 1.0]); d /= np.linalg.norm(d)
        ids = sorted(rng.choice(6, int(rng.integers(3, 7)), replace=False).tolist())
        inf.append(len(obs))
        obs.append((ids, [project(P[c], np.append(d, 0.0)) for c in ids]))
    return Problem(obs, np.stack(P), np.stack(Cs), tags={"far": far, "infinite": inf})


LONG_LIST_COUNTS = (3, 4, 31, 32, 33, 2000)
LONGEST_LIST = 10 ** 4


def long_lists(seed=3):
    """Points with 3, 4, 31, 32, 33 and 2000 noisy observations (three of each) and one with 10^4, cameras drawn with repeats from a
    ring of 64: tag 'long'"""
    rng = np.random.default_rng(seed)
    K = np.array([[1200.0, 0, 960], [0, 1200.0, 540], [0, 0, 1]])
    ang = np.linspace(0, 2 * np.pi, 64, endpoint=False)
    Cs = np.stack([30 * np.cos(ang), 30 * np.sin(ang), 10 + 2 * np.sin(3 * ang)], 1)
    P = np.stack([projection(K, look_at(C, np.zeros(3)), C) for C in Cs])
    obs = []
    for m in [c for c in LONG_LIST_COUNTS for _ in range(3)] + [LONGEST_LIST]:
        X = rng.uniform(-5, 5, 3)
        ids = rng.integers(0, 64, m)
        h = np.einsum("nij,j->ni", P[ids], np.append(X, 1.0))
        obs.append((ids.tolist(), (h[:, :2] / h[:, 2:] + rng.normal(0, 0.5, (m, 2))).tolist()))
    return Problem(obs, P, Cs, tags={"long": list(range(len(obs)))})


def rank_deficient(seed=4):
    """Null spaces of two dimensions: one camera seen three to six times at one pixel, and two cameras with the same matrix under two
    ids: tag 'null2'; plus two regular points: tag 'regular'"""
    rng = np.random.default_rng(seed)
    K = np.array([[1200.0, 0, 960], [0, 1200.0, 540], [0, 0, 1]])
    Cs = [np.array([20.0, 0, 5]), np.array([0, 20.0, 5]), np.array([-20.0, 0, 5])]
    P = [projection(K, look_at(C, np.zeros(3)), C) for C in Cs]
    P.append(P[0].copy())                                  # camera 3 is camera 0 again
    obs, null2 = [], []
    for m in (3, 4, 6):
        X = rng.uniform(-3, 3, 3)
        null2.append(len(obs))
        obs.append(([1] * m, [project(P[1], np.append(X, 1.0))] * m))
        null2.append(len(obs))
        obs.append(([0, 3, 0][:m] + [3] * (m - 3), [project(P[0], np.append(X, 1.0)) + rng.normal(0, 0.3, 2)] * m))
    regular = []
    for _ in range(2):
        X = rng.uniform(-3, 3, 3)
        regular.append(len(obs))
        obs.append(([0, 1, 2], [project(P[c], np.append(X, 1.0)) for c in (0, 1, 2)]))
    return Problem(obs, np.stack(P), np.stack(Cs + [Cs[0]]), tags={"null2": null2, "regular": regular})


def non_finite(seed=5):
    """Regular points and points with one non-finite input: NaN or +-Inf in x or y, or a camera whose matrix holds NaN or Inf (cameras
    4 and 5): tags 'nonfinite' and 'regular'"""
    rng = np.random.default_rng(seed)
    K = np.array([[1200.0, 0, 960], [0, 1200.0, 540], [0, 0, 1]])
    Cs = [np.array([25 * np.cos(a), 25 * np.sin(a), 6.0]) for a in np.linspace(0, 2 * np.pi, 6, endpoint=False)]
    P = np.stack([projection(K, look_at(C, np.zeros(3)), C) for C in Cs])
    P[4, 1, 2] = np.nan
    P[5, 2, 3] = np.inf
    obs, bad, regular = [], [], []
    for k in range(48):
        X = rng.uniform(-3, 3, 3)
        ids = sorted(rng.choice(4, 3, replace=False).tolist())
        xy = [project(P[c], np.append(X, 1.0)) + rng.normal(0, 0.3, 2) for c in ids]
        kind = k % 8
        if kind == 0:
            regular.append(len(obs))
        elif kind <= 5:
            v = (np.nan, np.inf, -np.inf, np.nan, np.inf)[kind - 1]
            xy[int(rng.integers(0, 3))][(kind - 1) % 2] = v
            bad.append(len(obs))
        else:
            ids[1] = 4 if kind == 6 else 5
            xy[1] = np.array([900.0, 500.0])
            bad.append(len(obs))
        obs.append((ids, xy))
    return Problem(obs, P, np.stack(Cs), tags={"nonfinite": bad, "regular": regular})


def ring_points(n, lo, hi, ncam=64, seed=6, noise=0.5):
    """n points in [-5, 5]^3 with lo..hi noisy observations each by cameras drawn with repeats from ncam on a ring of radius 30
    (f = 1200 px); camera i has the matrix of camera i % 64"""
    rng = np.random.default_rng(seed)
    K = np.array([[1200.0, 0, 960], [0, 1200.0, 540], [0, 0, 1]])
    ang = np.linspace(0, 2 * np.pi, 64, endpoint=False)
    base = np.stack([projection(K, look_at(C, np.zeros(3)), C) for C in np.stack([30 * np.cos(ang), 30 * np.sin(ang), 10 + 2 * np.sin(3 * ang)], 1)])
    P = base[np.arange(ncam) % 64]
    X = rng.uniform(-5, 5, (n, 3))
    cnt = rng.integers(lo, hi + 1, n)
    p = Problem([], P)
    p.ptr = np.zeros(n + 1, np.int64)
    p.ptr[1:] = np.cumsum(cnt)
    m = int(p.ptr[-1])
    p.cam = (rng.integers(0, 64, m) + 64 * rng.integers(0, max(ncam // 64, 1), m)).astype(np.int32) % ncam
    h = np.einsum("nij,nj->ni", P[p.cam], np.hstack([np.repeat(X, cnt, 0), np.ones((m, 1))]))
    p.xy = h[:, :2] / h[:, 2:] + rng.normal(0, noise, (m, 2))
    return p


# ---------------------------------------------------------------------------------------------- median-depth problems
MEDIAN_CAMERA_COUNTS = (499, 500, 501, 5000)
# both sides of the small and medium segment limits and of one block-radix tile, and one list of more than 10^5 keys
MEDIAN_LIST_LENGTHS = (0, 1, 2, CUB_SMALL_MAX - 1, CUB_SMALL_MAX, CUB_SMALL_MAX + 1, CUB_MEDIUM_MAX - 1, CUB_MEDIUM_MAX, CUB_MEDIUM_MAX + 1,
                       CUB_LARGE_TILE - 1, CUB_LARGE_TILE, CUB_LARGE_TILE + 1, 100_003)


def median_lists(n_cams, n_points=20000, seed=0):
    """n_cams cameras whose first lists have the lengths MEDIAN_LIST_LENGTHS and the rest 0-150 entries, ids with repeats into
    n_points points of which about 80 % are valid: (lptr, lpts, X, valid, centres)"""
    rng = np.random.default_rng(seed + n_cams)
    X = rng.uniform(-50, 50, (n_points, 3))
    valid = (rng.uniform(size=n_points) > 0.2).astype(np.int32)
    Cs = rng.uniform(-10, 10, (n_cams, 3))
    sizes = rng.integers(0, 151, n_cams)
    k = min(n_cams, len(MEDIAN_LIST_LENGTHS))
    sizes[:k] = MEDIAN_LIST_LENGTHS[:k]
    lptr = np.zeros(n_cams + 1, np.int64)
    lptr[1:] = np.cumsum(sizes)
    return lptr, rng.integers(0, n_points, int(lptr[-1])).astype(np.int32), X, valid, Cs


def median_edges():
    """lists whose depths tie, sit one float ulp apart, are +0, +inf or overflow float (1e39) or double (1e200) to inf, and lists
    with no valid point; every camera at the origin except the last: (lptr, lpts, X, valid, centres, names)"""
    pts, lists, names = [], [], []
    def add(p):
        pts.append(p)
        return len(pts) - 1
    invalid = [add((1.0, 2.0, 3.0)) for _ in range(3)]
    r = 7.25
    ties = [add(v) for v in ((r, 0, 0), (0, r, 0), (0, 0, r), (-r, 0, 0), (0, -r, 0), (0, 0, -r))]
    lists.append(("equal", ties * 200 + invalid))
    u = [np.float32(1000.0)]
    for _ in range(40):
        u.append(np.nextafter(u[-1], np.float32(np.inf)))
    one_ulp = [add((float(v), 0.0, 0.0)) for v in u]
    lists.append(("one ulp apart", one_ulp[::-1] + one_ulp[::3]))
    zero, inf = add((0.0, 0.0, 0.0)), add((np.inf, 0.0, 0.0))
    lists.append(("+0 and +inf", [zero, inf, zero, inf, inf] + ties[:2]))
    lists.append(("only +0", [zero] * 5))
    lists.append(("only +inf", [inf] * 4 + invalid))
    f_over, d_over = add((1e39, 0.0, 0.0)), add((1e200, -1e200, 0.0))
    lists.append(("overflow", [f_over, d_over, ties[0], f_over]))
    lists.append(("only invalid", invalid * 50))
    lists.append(("empty", []))
    lists.append(("other centre", ties + one_ulp + [zero, inf]))
    X = np.array(pts, np.float64)
    valid = np.ones(len(X), np.int32)
    valid[invalid] = 0
    lptr = np.zeros(len(lists) + 1, np.int64)
    lptr[1:] = np.cumsum([len(l) for _, l in lists])
    Cs = np.zeros((len(lists), 3))
    Cs[-1] = (0.5, -0.25, 3.0)
    return lptr, np.array([i for _, l in lists for i in l], np.int32), X, valid, Cs, [n for n, _ in lists]


def join_medians(a, b):
    """two median problems as one: b's cameras after a's, b's point ids after a's"""
    la, pa, Xa, va, Ca = a[:5]
    lb, pb, Xb, vb, Cb = b[:5]
    return (np.concatenate([la, lb[1:] + la[-1]]), np.concatenate([pa, pb + len(Xa)]).astype(np.int32), np.concatenate([Xa, Xb]),
            np.concatenate([va, vb]), np.concatenate([Ca, Cb]))


def median_sort_problem(n_cams, seed=0):
    """exactly n_cams cameras, so exactly n_cams segments for cub: the lists of median_lists, then the nine lists of median_edges"""
    edges = median_edges()
    return join_medians(median_lists(n_cams - (len(edges[0]) - 1), seed=seed), edges)
