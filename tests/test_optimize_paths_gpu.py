"""l3d_optimize_lines against the float64 restatement (tests/opt_model.py) and the CPU oracle on the problems built to reach every
step, failure and termination path of the bundling (tests/test_opt_model_cpu.py pins the oracle to the model on the same
problems), its determinism, a problem of the size timed in DESIGN.md, and its checks on the residual offsets.

The invalid problem pins the library's current rule only: a step whose 4x4 solve fails is "invalid", halves the radius and
recomputes the diagonal, and five in a row end the run with a failure.  Ceres may instead reject an evaluation whose residuals
or Jacobian are not finite, and may treat an invalid step like a rejected one (DESIGN.md §8f-4); that is not settled here.
Not tested: the minimum trust-region radius (1e-32), which no run reaches before a tolerance ends it."""
import ctypes as C
import math

import numpy as np
import pytest

from tests import opt_model as om
from tests.test_opt_model_cpu import ATOL_ALL, ATOL_FEW, MAX_ITERS, PROBLEMS, RTOL_COST, RTOL_COST0, assert_same_run, model, oracle_run, problem

pytestmark = pytest.mark.gpu


def run(ctx, pr, max_iter):
    return ctx.optimize_lines(pr["p1p2"], pr["res_ptr"], pr["res_cam"], pr["res_xy"], pr["cams"], max_iter)


@pytest.mark.parametrize("max_iter", MAX_ITERS)
@pytest.mark.parametrize("name", PROBLEMS)
def test_gpu_matches_model_and_oracle(gpu_ctx, oracle, name, max_iter):
    out, valid, summ = run(gpu_ctx, problem(name), max_iter)
    atol = ATOL_FEW if max_iter <= 3 else ATOL_ALL
    assert_same_run(name, max_iter, out, valid, summ, atol)
    o, ov, osumm = oracle_run(name, max_iter)
    assert list(summ[[0, 3, 4, 5]]) == list(osumm[[0, 3, 4, 5]]) and np.array_equal(valid, ov)
    keep = valid == 1
    np.testing.assert_allclose(out[keep], o[keep], rtol=0, atol=atol)
    np.testing.assert_array_equal(out[~keep], o[~keep])


@pytest.mark.parametrize("n", om.SIZES)
def test_costs_are_the_exact_sums_of_the_model_line_costs(gpu_ctx, n):
    """k_opt_reduce's fixed-order sums against math.fsum of the model's per-line costs, across the 128-thread block and the
    1024-wide reduction boundaries"""
    name = f"sizes_{n}"
    m = model(name, 250)
    _, _, s0 = run(gpu_ctx, problem(name), 0)
    c0 = math.fsum(m["line_cost0"].tolist())
    assert abs(s0[1] - c0) <= RTOL_COST0 * c0 and s0[2] == s0[1]
    _, _, s = run(gpu_ctx, problem(name), 250)
    assert abs(s[1] - c0) <= RTOL_COST0 * c0
    assert abs(s[2] - math.fsum(m["line_cost"].tolist())) <= RTOL_COST * c0


def test_repeatable_and_independent_of_earlier_calls(gpu_ctx):
    """bit-identical on a repeat; a large problem first leaves nothing behind in the reused device buffers (diagonal, candidate
    point, partial sums); the output may alias the input"""
    from line3dpp_b200 import capi
    small, big = problem("outliers"), problem("sizes_4097")
    a = run(gpu_ctx, small, 250)
    b = run(gpu_ctx, small, 250)
    for u, v in zip(a, b):
        assert np.array_equal(u.view(np.uint8), v.view(np.uint8))
    ctx = capi.Context(0)
    try:
        fresh = run(ctx, small, 250)
        run(ctx, big, 250)
        after = run(ctx, small, 250)
        p = np.ascontiguousarray(small["p1p2"], np.float64).copy()
        ptr = np.ascontiguousarray(small["res_ptr"], np.int64); rc = np.ascontiguousarray(small["res_cam"], np.int32)
        xy = np.ascontiguousarray(small["res_xy"], np.float64); cams = np.ascontiguousarray(small["cams"], np.float64)
        valid = np.zeros(len(p), np.int32); summ = np.zeros(8)
        ptr_of = lambda x: x.ctypes.data_as(C.c_void_p)                            # noqa: E731
        rcode = ctx.L.l3d_optimize_lines(ctx.h, len(p), ptr_of(p), ptr_of(ptr), ptr_of(rc), ptr_of(xy), len(cams), ptr_of(cams), 250,
                                         ptr_of(p), ptr_of(valid), ptr_of(summ))
        assert rcode == 0
    finally:
        ctx.close()
    for u, v in zip(fresh, after):
        assert np.array_equal(u.view(np.uint8), v.view(np.uint8))
    for u, v in zip(fresh, a):
        assert np.array_equal(u.view(np.uint8), v.view(np.uint8))
    assert np.array_equal(p.view(np.uint8), a[0].view(np.uint8)) and np.array_equal(valid, a[1]) and np.array_equal(summ, a[2])


def test_at_the_size_timed_in_design_md(gpu_ctx, oracle):
    """about 100 000 lines and 700 000 residuals (DESIGN.md times 99 560 lines, 704 120 residuals) against the oracle, 3 iterations"""
    pr = om._scene(np.random.default_rng(77), np.random.default_rng(78).integers(1, 13, 100_000), ncam=40)
    assert 650_000 < pr["res_ptr"][-1] < 750_000
    out, valid, summ = run(gpu_ctx, pr, 3)
    o, ov, os_ = oracle.optimize_lines(oracle.lib().orc_optimize_lines, pr["p1p2"], pr["res_ptr"], pr["res_cam"], pr["res_xy"], pr["cams"], 3)
    assert list(summ[[0, 3, 4, 5]]) == list(os_[[0, 3, 4, 5]]) and summ[5] == 100_000 and np.array_equal(valid, ov)
    assert abs(summ[1] - os_[1]) <= RTOL_COST0 * os_[1] and abs(summ[2] - os_[2]) <= RTOL_COST * os_[1]
    np.testing.assert_allclose(out, o, rtol=0, atol=ATOL_FEW)


def test_bad_residual_offsets_are_rejected(gpu_ctx):
    from line3dpp_b200 import capi
    pr = problem("sizes_129")
    for ptr, what in ((pr["res_ptr"] + 1, "res_ptr[0] must be 0"), (np.r_[pr["res_ptr"][:50], pr["res_ptr"][50:] - 10], "must not decrease")):
        with pytest.raises(capi.L3DError, match=what.replace("[", r"\[").replace("]", r"\]")):
            gpu_ctx.optimize_lines(pr["p1p2"], ptr, pr["res_cam"], pr["res_xy"], pr["cams"], 10)
    out, valid, summ = run(gpu_ctx, pr, 250)                       # the context is still usable
    assert_same_run("sizes_129", 250, out, valid, summ, ATOL_ALL)
