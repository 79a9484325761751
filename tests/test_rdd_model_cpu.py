"""The CPU oracle's diffusion (orc_rdd_f32_iters) against the float64 restatement (tests/rdd_model.py) on graphs built to reach
every walk length, padding, clamp and missing-transpose path of the diffusion kernels, and what each graph reaches.  The GPU side
(l3d_rdd bit for bit against the oracle on the same graphs) is tests/test_rdd_gpu.py."""
import functools

import numpy as np
import pytest

from tests import rdd_model as rm
from tests import util

# Worst deviation of the float32 oracle from the float64 model, relative to the model, over the entries above the clamp
# (iters 1, 2, 10, 11): 5.6e-5 on tiny_weights at 11 iterations (sums of values spread over 30 decades), at most 1.0e-5 on every
# other graph (hubs, 10 iterations: walks of thousands of values).  Entries at or below EPS on either side: measured 0, bound 1e-12.
RTOL = 1e-4
ATOL_CLAMP = 1e-12
ITERS = (1, 2, 10)


@functools.lru_cache(maxsize=None)
def oracle_rdd(name, iters):
    from oracle import pyoracle as po
    n, ei, ej, ew = rm.BUILDERS[name]()
    oi, oj, ow, _ = po.rdd(None, ei, ej, ew, n, iters=iters)
    return oi, oj, ow


@functools.lru_cache(maxsize=None)
def f64_trace(name, iters):
    return rm.rdd_f64_trace(*rm.BUILDERS[name](), iters)


def assert_close_to_f64(w32, w64):
    """w32 (float32 result) within RTOL of w64 where both are above EPS, within ATOL_CLAMP where either is at or below it"""
    w32 = np.asarray(w32, np.float64)
    clamp = (w64 <= rm.EPS) | (w32 <= rm.EPS)
    err = np.abs(w32 - w64)
    assert err[clamp].max(initial=0.0) <= ATOL_CLAMP
    rel = err[~clamp] / w64[~clamp]
    assert rel.max(initial=0.0) <= RTOL, (rel.max(), int(np.argmax(rel)))


@pytest.mark.parametrize("iters", ITERS)
@pytest.mark.parametrize("name", list(rm.BUILDERS))
def test_oracle_matches_f64_model(oracle, name, iters):
    oi, oj, ow = oracle_rdd(name, iters)
    mi, mj, ws, _ = f64_trace(name, max(ITERS))
    assert np.array_equal(oi, mi) and np.array_equal(oj, mj)
    assert_close_to_f64(ow, ws[iters - 1])


@pytest.mark.parametrize("name", list(rm.BUILDERS))
def test_oracle_iters_10_is_orc_rdd_f32(oracle, name):
    n, ei, ej, ew = rm.BUILDERS[name]()
    ci, cj, cw, _ = oracle.rdd(oracle.lib().orc_rdd_f32, ei, ej, ew, n)
    oi, oj, ow = oracle_rdd(name, 10)
    assert np.array_equal(ci, oi) and np.array_equal(cj, oj) and np.array_equal(util.bits(cw), util.bits(ow))


def _every_id_has_row_and_column(n, ei, ej):
    return np.all(np.bincount(ei, minlength=n) > 0) and np.all(np.bincount(ej, minlength=n) > 0)


@pytest.mark.parametrize("name", list(rm.BUILDERS))
def test_graph_reaches_its_paths(name):
    n, ei, ej, ew = rm.BUILDERS[name]()
    cov = rm.coverage(n, ei, ej)
    hist = cov["walk_hist"]
    n4 = 2 * ((cov["rowlen"] + 7) // 8)                  # float4 per padded row: <= 4 takes k_rdd_normalize_q's v0 path
    stats = f64_trace(name, max(ITERS))[3]
    # the verbatim reference reads start index -1 for an id without entries: every graph it is compared on has none
    assert _every_id_has_row_and_column(n, ei, ej) == (name != "isolated")
    if name == "ladder":
        assert all(L < len(hist) and hist[L] > 0 for L in range(1, 67))     # n8 = 1..9, incl. 7/8/9, 15/16/17, 24/25
        assert set(range(2, 21, 2)) <= set(n4.tolist())                   # both normalisation paths, every trip count
        assert cov["no_transpose"] == 0 and stats["sum_clamps"] == 0
    elif name == "hubs":
        assert cov["longest_walk"] > 1000
        rl = cov["rowlen"]
        hub = np.flatnonzero(rl > 1000)
        assert len(hub) == 4 and n - 1 in hub and {0, 7} <= set((hub % 8).tolist())
        for h in hub[hub < n - 1]:                                          # a hub row beside seven short rows in one warp
            warp = np.arange(h - h % 8, h - h % 8 + 8)
            assert np.all(rl[warp[warp != h]] <= 16)
        assert n % 8 and n % 64
    elif name == "tiny_weights":
        assert stats["sum_clamps_felt"] > 0 and stats["step_clamps"] > 0 and stats["subnormal_products"] > 0
        assert np.any(ew == 0) and ew[ew > 0].min() < 1e-29
    elif name == "asymmetric":
        assert 0.08 < cov["no_transpose"] / len(ei) < 0.12 and stats["no_transpose"] == cov["no_transpose"]
    elif name == "isolated":
        assert cov["empty_inside"] >= 64 + 3 and cov["after_last"] > 0
    elif name == "affinity_like":
        assert n >= 200000 and len(ei) >= 4_000_000
        assert (4 * n4.astype(np.int64)).sum() > 2 ** 22                  # padded slot offsets beyond 2^22 floats
    elif name == "tiny":
        assert n == 2 and len(ei) == 2
