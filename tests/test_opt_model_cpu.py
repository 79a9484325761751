"""The CPU oracle's bundling (orc_optimize_lines) against the float64 restatement (tests/opt_model.py) on problems built to reach
every step, failure and termination path of the trust-region minimiser, and what each problem reaches.  The GPU side
(l3d_optimize_lines against both on the same problems) is tests/test_optimize_paths_gpu.py.

Not tested: the minimum trust-region radius (1e-32).  The radius shrinks only on rejected or invalid steps, and the parameter
or function tolerance ends a run long before 1e-32; the rule is kept in the model."""
import functools

import numpy as np
import pytest

from tests import opt_model as om

PROBLEMS = list(om.KINDS) + [f"sizes_{n}" for n in om.SIZES]
MAX_ITERS = (0, 1, 2, 3, 250)
# Worst end-point gap between the oracle and the model on the lines both keep: 1.5e-6 scene units within 3 iterations (parallel:
# acos' ~ 1 / sqrt(1 - dot^2) amplifies the rounding of the first step next to |dot| == 1), 4.5e-6 at convergence (sizes_4097,
# 26 iterations), at most 2.2e-7 on every other problem within 3 iterations.
ATOL_FEW, ATOL_ALL = 5e-6, 2e-5
# Costs: the initial cost within 4e-14 of itself relative (summation order), the final cost within 1.2e-10 of the initial cost
# (sizes_1024: two trajectories that differ by rounding).  converged_step's cost (1e-13) is itself rounding: 3.4e-20 apart, so a
# floor of 1e-21 per residual is allowed on top.
RTOL_COST0, RTOL_COST, ATOL_COST_PER_RES = 1e-12, 1e-9, 1e-21


@functools.lru_cache(maxsize=None)
def problem(name):
    return om.make_problem(name)


@functools.lru_cache(maxsize=None)
def model(name, max_iter):
    return om.optimize(**problem(name), max_iter=max_iter)


@functools.lru_cache(maxsize=None)
def oracle_run(name, max_iter):
    from oracle import pyoracle as po
    pr = problem(name)
    return po.optimize_lines(po.lib().orc_optimize_lines, pr["p1p2"], pr["res_ptr"], pr["res_cam"], pr["res_xy"], pr["cams"], max_iter)


def assert_same_run(name, max_iter, out, valid, summ, atol):
    """one run (end points, valid flags, summary) against the model's"""
    m = model(name, max_iter)
    ms = m["summary"]
    assert list(summ[[0, 3, 4, 5]]) == list(ms[[0, 3, 4, 5]]), (summ, ms)     # iterations, termination, accepted steps, free lines
    assert np.array_equal(valid, m["valid"])
    floor = ATOL_COST_PER_RES * problem(name)["res_ptr"][-1]
    if np.isfinite(ms[1]):
        assert abs(summ[1] - ms[1]) <= RTOL_COST0 * abs(ms[1]) + floor, (summ[1], ms[1])
        assert abs(summ[2] - ms[2]) <= RTOL_COST * abs(ms[1]) + floor, (summ[2], ms[2])
    else:
        assert summ[1] == ms[1] and summ[2] == ms[2]
    # final trust-region radius: its update divides two nearly cancelling cost changes; worst measured 7.3e-5 relative (sizes_127)
    assert abs(summ[6] - ms[6]) <= 1e-2 * ms[6], (summ[6], ms[6])
    keep = m["valid"] == 1
    np.testing.assert_allclose(out[keep], m["p1p2_out"][keep], rtol=0, atol=atol)
    np.testing.assert_array_equal(out[~keep], m["p1p2_out"][~keep])       # old end points, NaN included


@pytest.mark.parametrize("max_iter", MAX_ITERS)
@pytest.mark.parametrize("name", PROBLEMS)
def test_oracle_matches_f64_model(oracle, name, max_iter):
    out, valid, summ = oracle_run(name, max_iter)
    assert_same_run(name, max_iter, out, valid, summ, ATOL_FEW if max_iter <= 3 else ATOL_ALL)


def test_complex_step_gradient_matches_central_differences_of_np_cost():
    """the model's robustified gradient J'r (complex step) against central differences of tests/test_cpu.py's _np_cost, an
    independent restatement of the cost of one line; lines from the noisy, outliers and flipped problems"""
    from tests.test_cpu import _np_cost
    checked = 0
    for name in ("noisy", "outliers", "flipped"):
        pr = problem(name)
        P = om._Problem(**pr)
        x, ok = om.cayley_from_segments(P.p)
        free = ok & (np.diff(P.ptr) > 0)
        cost, failed, g, _ = om._evaluate(P, free, x, True, None)
        assert not failed.any()
        for i in range(0, P.L, max(1, P.L // 12)):
            r0, r1 = P.ptr[i], P.ptr[i + 1]
            rc, xy = P.rc[r0:r1], P.xy[r0:r1]
            assert _np_cost(x[i], P.cams, rc, xy) == pytest.approx(cost[i], rel=1e-12)
            fd = np.empty(4)
            for k in range(4):
                h = 1e-6 * max(1.0, abs(x[i, k]))
                xp, xm = x[i].copy(), x[i].copy()
                xp[k] += h; xm[k] -= h
                fd[k] = (_np_cost(xp, P.cams, rc, xy) - _np_cost(xm, P.cams, rc, xy)) / (2 * h)
            np.testing.assert_allclose(g[i], fd, rtol=1e-5, atol=1e-6 * np.abs(g[i]).max())
            checked += 1
    assert checked >= 30


def test_conversions_round_trip():
    """Pluecker -> Cayley -> end points gives the same 3D line (unit length around the old mid point) on every dominant axis"""
    rng = np.random.default_rng(5)
    ctr = rng.uniform(-3, 3, (300, 3))
    d = rng.normal(size=(300, 3))
    d[:100, 0] = 10.0; d[100:200, 1] = -10.0; d[200:, 2] = 10.0      # x, y and z dominant
    p = np.concatenate([ctr - d, ctr + d], 1)
    x, ok = om.cayley_from_segments(p)
    out, valid, axis = om.segments_from_cayley(x, p)
    assert ok.all() and valid.all() and set(axis[:100]) == {0} and set(axis[100:200]) == {1} and set(axis[200:]) == {2}
    u = d / np.linalg.norm(d, axis=1, keepdims=True)
    v = (out[:, :3] - out[:, 3:]) / 2
    np.testing.assert_allclose(np.abs((v * u).sum(1)), 1.0, atol=1e-12)
    w = out[:, :3] - ctr                                            # the new points lie on the old line
    np.testing.assert_allclose(np.linalg.norm(w - (w * u).sum(1, keepdims=True) * u, axis=1), 0.0, atol=1e-11)


def test_each_problem_reaches_its_path():
    runs = {name: model(name, 250) for name in PROBLEMS}
    stops = {name: r["stop"] for name, r in runs.items()}

    r = runs["noisy"]
    assert r["stop"] == "function tolerance" and r["steps"]["accepted"] > 3 and r["steps"]["rejected"] > 0
    assert np.diff(problem("noisy")["res_ptr"]).max() == 1000
    assert {0, 1, 2} <= set(r["axis"])                              # all three dominant-axis cases of the write-back
    t = runs["outliers"]["tally0"]
    assert t["huber_linear"] > 0.2 * t["huber_quadratic"] > 0
    t = runs["flipped"]["tally0"]
    assert t["angle_flipped"] > 0.3 * (t["angle_direct"] + t["angle_flipped"])
    t = runs["parallel"]["tally0"]                                  # |dot| == 1 on every block at the start, then the run moves on
    assert t["angle_nonfinite"] == problem("parallel")["res_ptr"][-1] and t["angle_direct"] == t["angle_flipped"] == 0
    assert runs["parallel"]["steps"]["accepted"] > 3 and runs["parallel"]["tally"]["angle_direct"] > 0

    r = runs["converged_zero"]                                      # residuals and gradient exactly 0: stop at iteration zero
    assert r["stop"] == "gradient tolerance" and r["summary"][0] == 0 and r["summary"][1] == 0.0
    r = runs["converged_step"]                                      # gradient above 1e-10, first step below the parameter tolerance
    assert r["stop"] == "parameter tolerance" and r["summary"][0] == 1 and r["summary"][1] > 0
    assert {"gradient tolerance", "parameter tolerance", "function tolerance"} <= set(stops.values())

    r, pr = runs["mixed_free"], problem("mixed_free")
    i = np.arange(len(pr["p1p2"]))
    counts = np.diff(pr["res_ptr"])
    assert np.array_equal(r["free"], (i % 7 != 0) & (i % 7 != 3)) and (counts[i % 7 == 3] > 0).all()
    assert np.array_equal(r["valid"] == 0, (i % 7 == 3) | (i % 14 == 7))
    kept = (i % 7 == 3) | (i % 14 == 7)
    assert np.array_equal(r["p1p2_out"][kept], pr["p1p2"][kept], equal_nan=True)
    assert r["stop"] == "function tolerance" and r["steps"]["accepted"] > 0

    for name, bad in (("through_origin", 11), ("through_camera", 9), ("zero_length", 6)):
        r, pr = runs[name], problem(name)
        assert r["stop"] == "initial evaluation failed" and list(r["summary"][[0, 1, 2, 3, 4]]) == [0, 0, 0, 2, 0]
        assert r["free"].all()                                      # the failing line is free: nothing is held constant
        p, out = pr["p1p2"], r["p1p2_out"]
        others = np.arange(len(p)) != bad
        mid = 0.5 * (p[:, :3] + p[:, 3:])                           # every other line: unit length around its old mid point
        np.testing.assert_allclose(np.linalg.norm(out[others, :3] - out[others, 3:], axis=1), 2.0, atol=1e-12)
        np.testing.assert_allclose(0.5 * (out[others, :3] + out[others, 3:]) - mid[others], 0.0, atol=1e-9)
    assert np.array_equal(runs["through_origin"]["p1p2_out"][11], problem("through_origin")["p1p2"][11])     # omega = 0: kept
    assert runs["zero_length"]["valid"][6] == 0 and runs["through_origin"]["x"][11, 0] == 0.0

    r = runs["invalid"]                                             # J'J overflows: five invalid steps and a failure
    assert r["stop"] == "invalid steps" and r["steps"] == dict(accepted=0, rejected=0, invalid=5) and r["summary"][3] == 2
    assert np.isfinite(r["summary"][1]) and not np.isfinite(r["H0"][4]).all() and np.isfinite(r["H0"][np.arange(40) != 4]).all()

    for n in om.SIZES:
        assert runs[f"sizes_{n}"]["summary"][5] == n and runs[f"sizes_{n}"]["summary"][3] == 0
