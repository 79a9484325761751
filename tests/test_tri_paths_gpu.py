"""l3d_triangulate_points and l3d_median_depths (DESIGN.md §6b) against the extended-precision model of tests/tri_model.py on problems
that reach every path: Pix4D coordinate scales, kappa up to 1e14, points at and near infinity, lists of 3 to 10^4 observations, null
spaces of two dimensions, non-finite input, camera matrices in shared and in global memory, a grid that strides, every partition of
cub's segmented sort, device addresses, and buffers reused across calls.

Every triangulated point with finite input is held to ||X - X*|| <= C_BOUND 2^-52 kappa sqrt(1 + ||X*||^2) (1 + ||X*||), and its valid
flag to the model's wherever ||X*|| is farther than that bound from L3D_EPS.  Median depths are exact."""
import numpy as np
import pytest
import torch

from line3dpp_b200 import capi
from tests import tri_model as tm

pytestmark = pytest.mark.gpu

# One constant for the whole file: 9x the largest ratio ||X - X*|| / (2^-52 kappa sqrt(1 + ||X*||^2) (1 + ||X*||)) measured over these
# problems, 1.33, on one H100 80GB HBM3 (700 W power limit); the largest direction ratio of the distant points there is 0.0056.  The
# ratios do not depend on the clock: the kernel is deterministic.
C_BOUND = 12.0


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _check(p, m, X, valid):
    """the bound on every bounded point, the model's flag wherever it is decided, and the reference's rule everywhere: X = 0 and
    invalid without three observations of known cameras, otherwise valid == (|X| > L3D_EPS) (NaN invalid, +-Inf valid)"""
    r = m.ratio(X)
    worst = np.nanmax(r) if np.isfinite(r).any() else 0.0
    print(f"max bound ratio {worst:.3e} over {np.isfinite(r).sum()} points ({m.exact.sum()} exact)")
    assert worst <= C_BOUND, (worst, int(np.nanargmax(r)))
    dec = m.flag_decidable(C_BOUND)
    assert np.array_equal(valid[dec], m.valid[dec]), np.flatnonzero(valid[dec] != m.valid[dec])
    with np.errstate(invalid="ignore", over="ignore"):
        nrm = np.sqrt(X[:, 0] * X[:, 0] + X[:, 1] * X[:, 1] + X[:, 2] * X[:, 2])
    assert np.array_equal(valid, (m.enough & (nrm > tm.L3D_EPS)).astype(np.int32))
    assert not X[~m.enough].any()
    return worst


def _run(ctx, p, **kw):
    m = tm.Model(p.ptr, p.cam, p.xy, p.P, special=p.special(), null2=p.tags.get("null2", ()), **kw)
    X, valid = ctx.triangulate_points(p.ptr, p.cam, p.xy, p.P)
    _check(p, m, X, valid)
    return m, X, valid


# ---------------------------------------------------------------------------------------------- triangulation
def test_pix4d_scale_and_offset(ctx):
    """georeferenced coordinates (offsets near 5e6 m, f up to 8000 px, 4000 x 3000 images) and the same scene with the offset
    subtracted: each within the bound of its model, and the two within the sum of their bounds of each other"""
    world, local, Xt = tm.pix4d_scale(20000)
    mw, Xw, vw = _run(ctx, world, n_sample=300, n_worst=150)
    ml, Xl, vl = _run(ctx, local, n_sample=300, n_worst=150)
    seen3 = np.diff(world.ptr) >= 3
    both = (vw == 1) & (vl == 1)
    assert np.array_equal(vw, vl) and np.array_equal(both, seen3) and both.sum() > 0.7 * world.n
    off = world.centres[0] - local.centres[0]
    gap = np.linalg.norm((Xl + off) - Xw, axis=1)
    assert (gap[both] <= (mw.bound(C_BOUND) + ml.bound(C_BOUND))[both]).all()
    assert np.median(np.linalg.norm(Xw - Xt, axis=1)[both]) < 0.05                                   # the survey itself triangulates


def test_ill_conditioned(ctx):
    p = tm.ill_conditioned()
    m, _, _ = _run(ctx, p)
    assert m.kappa[p.tags["ill"]].max() > 1e12


def test_near_infinity(ctx):
    """|v.w| from 1e-3 to 0.  The bound on the position grows like ||X*||^2 and allows more than ||X*|| itself on these points, so it
    checks little here; the direction of X is held to its own bound, C_BOUND 2^-52 kappa 2 sqrt(1 + ||X*||^2) / ||X*||, wherever X is
    finite, and the reference's rule (+-Inf valid, NaN invalid) holds everywhere"""
    p = tm.near_infinity()
    m, X, valid = _run(ctx, p)
    far, inf = p.tags["far"], p.tags["infinite"]
    assert valid[far].all() and np.isfinite(m.X[far]).all()
    r = m.direction_ratio(X)
    assert np.isfinite(r[far]).all()
    worst = np.nanmax(r[far + inf])
    print(f"max direction ratio {worst:.3e} over {np.isfinite(r[far + inf]).sum()} points")
    assert worst <= C_BOUND, (worst, int(np.nanargmax(r)))


def test_long_observation_lists(ctx):
    _run(ctx, tm.long_lists())


def test_two_dimensional_null_space(ctx):
    """one camera seen repeatedly (or two ids of one matrix): X* is not unique, so X must be a null vector: ||A^T A v|| <= C eps ||A^T A||"""
    p = tm.rank_deficient()
    m, X, valid = _run(ctx, p)
    for i in p.tags["null2"]:
        b, e = p.ptr[i], p.ptr[i + 1]
        assert np.isfinite(X[i]).all()
        res = tm.residual_ratio(p.cam[b:e], p.xy[b:e], p.P, X[i])
        print(f"null-space residual {res / tm.EPS:.3e} eps")
        assert res <= C_BOUND * tm.EPS, i


def test_non_finite_input_leaves_other_points_alone(ctx):
    p = tm.non_finite()
    m, X, valid = _run(ctx, p)
    bad = p.tags["nonfinite"]
    assert not (valid[bad] & np.isnan(X[bad]).any(1)).any()
    keep = np.setdiff1d(np.arange(p.n), bad)
    cnt = np.diff(p.ptr)[keep]
    ptr = np.concatenate([[0], np.cumsum(cnt)])
    sel = np.concatenate([np.arange(p.ptr[i], p.ptr[i + 1]) for i in keep])
    X2, v2 = ctx.triangulate_points(ptr, p.cam[sel], p.xy[sel], p.P)
    assert np.array_equal(X2, X[keep]) and np.array_equal(v2, valid[keep])


def test_staged_and_global_cameras_with_a_strided_grid(ctx):
    """1024 cameras (exactly 96 KB of matrices, staged in shared memory) and the same problem with a 1025th camera (read from global
    memory), with more points than threads can be resident on the whole GPU, so the staged grid strides: bit-identical, and within the
    bound of the model"""
    wave = torch.cuda.get_device_properties(0).multi_processor_count * torch.cuda.get_device_properties(0).max_threads_per_multi_processor
    p = tm.ring_points(wave + 4099, 3, 6, ncam=1024, seed=21)
    assert p.P.nbytes == tm.tr_smem_max() and p.cam.max() == 1023
    m = tm.Model(p.ptr, p.cam, p.xy, p.P, n_sample=300, n_worst=100)
    X, valid = ctx.triangulate_points(p.ptr, p.cam, p.xy, p.P)
    _check(p, m, X, valid)
    X2, v2 = ctx.triangulate_points(p.ptr, p.cam, p.xy, np.concatenate([p.P, p.P[:1]]))
    assert np.array_equal(X, X2) and np.array_equal(valid, v2)
    assert valid[wave:].all()


def test_device_mode_unknown_camera(ctx):
    """on device addresses an observation of a camera outside [0, n_cams) makes only its own point invalid (X = 0); every other
    point is bit-identical to the host call"""
    p = tm.ring_points(3000, 3, 9, seed=22)
    X, valid = ctx.triangulate_points(p.ptr, p.cam, p.xy, p.P)
    cam = p.cam.copy()
    hit = [5, 700, 2999]
    cam[p.ptr[5]] = len(p.P)
    cam[p.ptr[700] + 2] = -1
    cam[p.ptr[3000] - 1] = 2 ** 31 - 1
    dp, dc, dx, dP = _dev(p.ptr), _dev(cam), _dev(p.xy), _dev(p.P.reshape(-1, 12))
    dX = torch.full((p.n, 3), 7.0, dtype=torch.float64, device="cuda")
    dv = torch.full((p.n,), 7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ctx.triangulate_points_device(p.n, dp.data_ptr(), dc.data_ptr(), dx.data_ptr(), len(p.P), dP.data_ptr(), dX.data_ptr(), dv.data_ptr())
    ctx.sync()
    Xd, vd = dX.cpu().numpy(), dv.cpu().numpy()
    assert (vd[hit] == 0).all() and not Xd[hit].any()
    rest = np.setdiff1d(np.arange(p.n), hit)
    assert np.array_equal(Xd[rest], X[rest]) and np.array_equal(vd[rest], valid[rest])


# ---------------------------------------------------------------------------------------------- median depths
def _same_medians(got, want):
    assert np.array_equal(got[0], want[0]), np.flatnonzero(got[0] != want[0])[:10]
    assert np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32)), np.flatnonzero(got[1].view(np.uint32) != want[1].view(np.uint32))[:10]


@pytest.mark.parametrize("n_cams", tm.MEDIAN_CAMERA_COUNTS)
def test_median_depths_every_sort_path(ctx, n_cams):
    """499 and 500 cameras (segments) take cub's unpartitioned kernel, 501 and 5000 its small, medium and large segments; the lists
    straddle each segment limit and one block-radix tile, and one holds more than 10^5 keys; the edge lists are among them"""
    prob = tm.median_sort_problem(n_cams)
    assert len(prob[0]) - 1 == n_cams
    _same_medians(ctx.median_depths(*prob), tm.median_model(*prob))


@pytest.mark.parametrize("pad", [0, 600])
def test_median_depths_edges(ctx, pad):
    """ties, depths one float ulp apart, +0, +inf, overflow to inf, lists without a valid point; alone and behind `pad` cameras with
    short lists (partitioned)"""
    edges = tm.median_edges()
    prob = edges[:5] if not pad else tm.join_medians(tm.median_lists(pad), edges)
    assert (len(prob[0]) - 1 > tm.CUB_PARTITIONING_THRESHOLD) == (pad > 0)
    got, want = ctx.median_depths(*prob), tm.median_model(*prob)
    _same_medians(got, want)
    names = edges[5]
    at = lambda name: (got[0][pad + names.index(name)], got[1][pad + names.index(name)])
    assert at("only invalid") == (0, 0) and at("overflow")[1] == np.inf and at("only +inf")[1] == np.inf


def _median_device(ctx, lptr, lpts, X, valid, Cs):
    d = [_dev(a) for a in (lptr, lpts, X, valid, Cs)]
    cnt = torch.full((len(lptr) - 1,), -1, dtype=torch.int32, device="cuda")
    med = torch.full((len(lptr) - 1,), -1.0, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    ctx.median_depths_device(len(lptr) - 1, d[0].data_ptr(), d[1].data_ptr(), len(X), d[2].data_ptr(), d[3].data_ptr(), d[4].data_ptr(),
                             cnt.data_ptr(), med.data_ptr())
    ctx.sync()
    return cnt.cpu().numpy(), med.cpu().numpy()


@pytest.mark.parametrize("n_cams", [499, 5000])
def test_median_depths_device_mode(ctx, n_cams):
    """device addresses: bit-identical to the host call; ids outside [0, n_points) count as invalid"""
    prob = tm.median_sort_problem(n_cams, seed=3)
    assert len(prob[0]) - 1 == n_cams
    _same_medians(_median_device(ctx, *prob), ctx.median_depths(*prob))
    lptr, lpts, X, valid, Cs = prob
    lpts = lpts.copy()
    rng = np.random.default_rng(n_cams)
    out = rng.choice(len(lpts), len(lpts) // 10, replace=False)
    lpts[out] = rng.choice(np.array([-1, -2 ** 31, len(X), len(X) + 1, 2 ** 31 - 1], np.int64), len(out)).astype(np.int32)
    got = _median_device(ctx, lptr, lpts, X, valid, Cs)
    _same_medians(got, tm.median_model(lptr, lpts, X, valid, Cs))
    assert (got[0] <= ctx.median_depths(*prob)[0]).all()


# ---------------------------------------------------------------------------------------------- buffer reuse
def test_buffers_reused_across_growing_and_shrinking_calls(ctx):
    """one context through small, large and small problems of both calls gives what fresh contexts give, and the medians are the
    model's"""
    tris = [tm.ring_points(n, 3, k, ncam=c, seed=n) for n, k, c in ((500, 4, 64), (60000, 12, 1500), (700, 5, 64), (40, 30, 8))]
    meds = [tm.join_medians(tm.median_lists(c, n_points=n), tm.median_edges()) for c, n in ((20, 500), (800, 30000), (10, 400))]
    shared = [(ctx.triangulate_points(p.ptr, p.cam, p.xy, p.P), ctx.median_depths(*q)) for p, q in zip(tris, meds + [meds[0]])]
    for (t, md), p, q in zip(shared, tris, meds + [meds[0]]):
        fresh = capi.Context(0)
        try:
            X, v = fresh.triangulate_points(p.ptr, p.cam, p.xy, p.P)
            assert np.array_equal(t[0], X) and np.array_equal(t[1], v)
            _same_medians(md, fresh.median_depths(*q))
            _same_medians(md, tm.median_model(*q))
        finally:
            fresh.close()
