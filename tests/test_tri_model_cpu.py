"""The triangulation and median-depth model of tests/tri_model.py against independent computations, and its problem builders
against the paths they are named for: the kappa range, the list lengths and camera counts on both sides of cub's segmented-sort
limits, the shared-memory staging limit.  No GPU."""
from fractions import Fraction

import numpy as np
import pytest

from tests import tri_model as tm


def _normal_matrix_fractions(cams, xy, P):
    A = [[Fraction(0)] * 4 for _ in range(4)]
    for c, (x, y) in zip(cams, xy):
        M = [Fraction(float(v)) for v in np.asarray(P[c], np.float64).ravel()]
        x, y = Fraction(float(x)), Fraction(float(y))
        r1 = [-M[4 + j] + y * M[8 + j] for j in range(4)]
        r2 = [M[j] - x * M[8 + j] for j in range(4)]
        for r in range(4):
            for k in range(4):
                A[r][k] += r1[r] * r1[k] + r2[r] * r2[k]
    return A


@pytest.mark.parametrize("problem", ["ring", "pix4d", "ill", "far"])
def test_normal_matrix_is_exact(problem):
    """A^T A from the integers equals the rational computation entry for entry"""
    p = {"ring": lambda: tm.ring_points(4, 3, 40), "pix4d": lambda: tm.pix4d_scale(4)[0], "ill": tm.ill_conditioned, "far": tm.near_infinity}[problem]()
    for i in range(min(p.n, 4)):
        b, e = p.ptr[i], p.ptr[i + 1]
        N, s = tm.normal_matrix_exact(p.cam[b:e], p.xy[b:e], p.P)
        F = _normal_matrix_fractions(p.cam[b:e], p.xy[b:e], p.P)
        assert all(Fraction(int(N[r, c]), 1 << s) == F[r][c] for r in range(4) for c in range(4))


def test_model_matches_eigh_when_well_conditioned():
    p = tm.ring_points(300, 3, 20, seed=11)
    m = tm.Model(p.ptr, p.cam, p.xy, p.P, special=range(p.n))
    assert m.exact.all() and (m.kappa < 1e4).all()
    Xn, kn = tm._numpy_model(p.ptr, p.cam, p.xy, p.P.reshape(-1, 12))
    assert np.abs(kn / m.kappa - 1).max() < 1e-6
    rel = np.linalg.norm(Xn - m.X, axis=1) / np.linalg.norm(m.X, axis=1)
    assert rel.max() < 1e-11, rel.max()


def test_model_point_is_the_null_vector():
    """noise-free observations: X* is the point itself, the smallest eigenvalue zero to the rounding of the projections"""
    p = tm.ill_conditioned()
    i = p.tags["ill"][0]                       # baseline 1e-1 of the depth, exact projections
    b, e = p.ptr[i], p.ptr[i + 1]
    X, lam, vw, kappa = tm.point_exact(p.cam[b:e], p.xy[b:e], p.P)
    assert lam[0] < 1e-20 * lam[3] and 0 < lam[1] and kappa < 1e5
    assert abs(np.linalg.norm(np.append(X, 1.0)) * vw - 1) < 1e-12


def test_median_model_is_sort_and_pick():
    lptr, lpts, X, valid, Cs, names = tm.median_edges()
    cnt, med = tm.median_model(lptr, lpts, X, valid, Cs)
    for c in range(len(names)):
        with np.errstate(over="ignore"):
            d = sorted(np.float32(np.linalg.norm(X[i] - Cs[c])) for i in lpts[lptr[c]:lptr[c + 1]] if valid[i])
        assert cnt[c] == len(d) and med[c] == (d[len(d) // 2] if d else 0), names[c]
    at = dict(zip(names, zip(cnt, med)))
    assert at["only invalid"] == (0, 0) and at["empty"] == (0, 0)
    assert at["only +0"] == (5, 0) and np.signbit(med[names.index("only +0")]) == 0
    assert at["only +inf"][1] == np.inf and at["overflow"][1] == np.inf
    d = X[lpts[lptr[1]:lptr[2]], 0].astype(np.float32)
    assert len(np.unique(d)) == 41 and np.all(np.diff(np.unique(d).view(np.uint32)) == 1)     # consecutive floats


# ---------------------------------------------------------------------------------------------- the builders reach their paths
def test_ill_conditioned_spans_kappa():
    p = tm.ill_conditioned()
    m = tm.Model(p.ptr, p.cam, p.xy, p.P, special=p.special())
    k = m.kappa[p.tags["ill"]]
    assert m.exact[p.tags["ill"]].all()
    assert k.min() < 1e4 and k.max() > 1e12, (k.min(), k.max())
    assert (np.histogram(np.log10(k), bins=range(2, 16))[0] > 0).sum() >= 10          # every decade in between


def test_near_infinity_reaches_zero_w():
    p = tm.near_infinity()
    m = tm.Model(p.ptr, p.cam, p.xy, p.P, special=p.special())
    vw = m.vw[p.tags["far"] + p.tags["infinite"]]
    assert vw.max() > 1e-4 and vw.min() < 1e-14
    assert (m.vw[p.tags["infinite"]] < 1e-12).all()


def test_long_lists_and_camera_counts():
    p = tm.long_lists()
    cnt = np.diff(p.ptr)[p.tags["long"]]
    assert set(tm.LONG_LIST_COUNTS) <= set(cnt.tolist()) and cnt.max() == tm.LONGEST_LIST
    # k_triangulate stages the camera matrices in shared memory up to TR_SMEM_MAX bytes: the 1024 cameras of the GPU test fill it
    # exactly and one more does not fit
    p = tm.ring_points(2000, 3, 6, ncam=1024, seed=21)
    assert p.P.nbytes == tm.tr_smem_max() and p.cam.max() == 1023 and np.concatenate([p.P, p.P[:1]]).nbytes > tm.tr_smem_max()


def test_rank_deficient_has_two_null_vectors():
    p = tm.rank_deficient()
    for i in p.tags["null2"]:
        b, e = p.ptr[i], p.ptr[i + 1]
        _, lam, _, kappa = tm.point_exact(p.cam[b:e], p.xy[b:e], p.P)
        assert abs(lam[1]) < 1e-60 * lam[3] and kappa > 1e50
        N, _ = tm.normal_matrix_exact(p.cam[b:e], p.xy[b:e], p.P)
        F = np.array([[Fraction(int(v)) for v in row] for row in N], dtype=object)
        assert _rank(F) == 2


def _rank(F):
    F = [list(r) for r in F]
    rank = 0
    for c in range(4):
        piv = next((r for r in range(rank, 4) if F[r][c] != 0), None)
        if piv is None:
            continue
        F[rank], F[piv] = F[piv], F[rank]
        for r in range(4):
            if r != rank and F[r][c] != 0:
                f = F[r][c] / F[rank][c]
                F[r] = [a - f * b for a, b in zip(F[r], F[rank])]
        rank += 1
    return rank


def test_non_finite_inputs_are_flagged():
    p = tm.non_finite()
    m = tm.Model(p.ptr, p.cam, p.xy, p.P, special=p.special())
    assert np.flatnonzero(m.nonfinite).tolist() == p.tags["nonfinite"]
    assert m.valid[p.tags["regular"]].all()
    assert {v for i in p.tags["nonfinite"] for v in p.xy[p.ptr[i]:p.ptr[i + 1]].ravel() if not np.isfinite(v)} >= {np.inf, -np.inf}
    assert np.isnan(p.xy).any() and np.isnan(p.P).any() and np.isinf(p.P).any()


def test_pix4d_scale_problem():
    world, local, Xt = tm.pix4d_scale(400)
    assert np.abs(world.centres).max() > 1e6 and np.abs(Xt).min(0)[:2].min() > 1e5
    assert world.focal.min() > 3000 and world.focal.max() < 8000
    assert np.array_equal(world.xy, local.xy) and np.array_equal(world.cam, local.cam)
    assert (world.xy >= -5).all() and (world.xy[:, 0] < 4005).all() and (world.xy[:, 1] < 3005).all()
    tilt = np.degrees(np.arccos(-world.P[:, 2, 2]))                                         # P[2, :3] is the viewing direction
    assert (tilt < 5).sum() >= 40 and (np.abs(tilt - 45) < 10).sum() >= 20                  # nadir and oblique views


def test_cub_limits_are_the_installed_ones():
    if not tm.cub_header_present():
        pytest.skip("no CUDA toolkit headers on this machine")
    assert tm.cub_limits() == (tm.CUB_PARTITIONING_THRESHOLD, tm.CUB_SMALL_MAX, tm.CUB_MEDIUM_MAX, tm.CUB_LARGE_TILE)


def test_median_problems_straddle_the_cub_limits():
    """the problems the GPU tests sort: as many segments as they claim, on both sides of the partitioning threshold, every one with
    lists on both sides of each segment-size limit; the multi-pass lists (one tile or more, and more than 10^5 keys) run unpartitioned
    too"""
    T = tm.CUB_PARTITIONING_THRESHOLD
    counts = tm.MEDIAN_CAMERA_COUNTS
    assert min(counts) < T and T in counts and any(T < c < 2 * T for c in counts) and max(counts) > 5 * T
    for n_cams in counts:
        lptr = tm.median_sort_problem(n_cams)[0]
        assert len(lptr) - 1 == n_cams
        sizes = set(np.diff(lptr).tolist())
        for limit in (tm.CUB_SMALL_MAX, tm.CUB_MEDIUM_MAX, tm.CUB_LARGE_TILE):
            assert {limit - 1, limit, limit + 1} <= sizes, (n_cams, limit)
        assert 0 in sizes and max(sizes) > 10 ** 5
        if n_cams <= T:
            assert max(sizes) >= tm.CUB_LARGE_TILE                                          # the unpartitioned multi-pass branch
    edges = tm.median_edges()
    assert len(edges[0]) - 1 <= T < len(tm.join_medians(tm.median_lists(600), edges)[0]) - 1   # the edge lists, alone and padded
