"""l3d_rdd and l3d_rdd_affinity on graphs that reach every walk, padding and clamp path of the diffusion kernels
(tests/rdd_model.py): bit for bit against the CPU oracle (orc_rdd_f32_iters) and the verbatim reference, within the stated
tolerance of the float64 model, independent of input order and of what the context computed before."""
import ctypes as C
import functools

import numpy as np
import pytest

from line3dpp_b200 import synth
from tests import rdd_model as rm
from tests import util
from tests.test_affinity_gpu import _scored_context, affinity_matrix
from tests.test_rdd_model_cpu import assert_close_to_f64, oracle_rdd

pytestmark = pytest.mark.gpu

ITERS = (1, 2, 10, 11)


@functools.lru_cache(maxsize=None)
def f64_trace(name):
    return rm.rdd_f64_trace(*rm.BUILDERS[name](), max(ITERS))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip((a[0], a[1], util.bits(a[2])), (b[0], b[1], util.bits(b[2]))))


@pytest.mark.parametrize("iters", ITERS)
@pytest.mark.parametrize("name", list(rm.BUILDERS))
def test_rdd_bit_exact_vs_oracle(gpu_ctx, oracle, name, iters):
    n, ei, ej, ew = rm.BUILDERS[name]()
    oi, oj, ow, _ = gpu_ctx.rdd(n, ei, ej, ew, iters)
    ci, cj, cw = oracle_rdd(name, iters)
    assert np.array_equal(oi, ci) and np.array_equal(oj, cj)
    assert np.array_equal(util.bits(ow), util.bits(cw))
    assert_close_to_f64(ow, f64_trace(name)[2][iters - 1])


@pytest.mark.parametrize("name", [b for b in rm.BUILDERS if b != "isolated"])     # an empty row is undefined in the reference
def test_rdd_bit_exact_vs_reference(gpu_ctx, ref_nofma, oracle, name):
    n, ei, ej, ew = rm.BUILDERS[name]()
    ri, rj, rw, _ = oracle.rdd(ref_nofma.ref_rdd, ei, ej, ew, n)
    assert _same(gpu_ctx.rdd(n, ei, ej, ew, 10)[:3], (ri, rj, rw))


@pytest.mark.parametrize("name", list(rm.BUILDERS))
def test_rdd_input_order_does_not_matter(gpu_ctx, name):
    n, ei, ej, ew = rm.BUILDERS[name]()
    perm = np.random.default_rng(len(ei)).permutation(len(ei))
    assert _same(gpu_ctx.rdd(n, ei[perm], ej[perm], ew[perm], 10)[:3], gpu_ctx.rdd(n, ei, ej, ew, 10)[:3])


def test_rdd_repeat_and_shrink_reuse_buffers(oracle):
    """the same call twice gives the same bytes; after a larger graph, a smaller one on the same context gives its own result (the
    context's buffers only grow: stale rows, pointers or padding of the larger graph must not leak into it)"""
    from line3dpp_b200 import capi
    ctx = capi.Context(0)
    try:
        small, large = rm.BUILDERS["hubs"](), rm.BUILDERS["affinity_like"]()
        first = ctx.rdd(*small, 10)[:3]
        assert _same(ctx.rdd(*small, 10)[:3], first)
        assert _same(ctx.rdd(*large, 10)[:3], oracle_rdd("affinity_like", 10))
        for name in ("hubs", "isolated", "tiny"):
            assert _same(ctx.rdd(*rm.BUILDERS[name](), 10)[:3], oracle_rdd(name, 10)), name
    finally:
        ctx.close()


@pytest.fixture(scope="module", params=["plain", "linked"])
def affinity_ctx(request):
    """the synthetic scenes of tests/test_affinity_gpu.py, without and with collinearity links, with their affinity matrix"""
    if request.param == "plain":
        ctx, med = _scored_context(synth.make_scene(14, 500, 31, "ring3"))
    else:
        ctx, med = _scored_context(synth.make_scene(12, 500, 93, "ring3", collinear=True))
        assert ctx.find_collinear(2.0, 0) > 1000
    ctx.L.l3d_rdd_affinity.restype = C.c_longlong
    ei, ej, ew, l2g = affinity_matrix(ctx, med)
    yield ctx, ei, ej, ew, len(l2g)
    ctx.close()


@pytest.mark.parametrize("iters", [1, 10])
def test_rdd_affinity_is_rdd_then_min_with_transpose(affinity_ctx, iters):
    """l3d_rdd_affinity == l3d_rdd on the CLEdge list l3d_affinity_matrix returned, then performRDD's min(w12, w21) per entry"""
    ctx, ei, ej, ew, num_ids = affinity_ctx
    nE = len(ei)
    assert nE > 1000
    oi, oj, ow = np.zeros(nE, np.int32), np.zeros(nE, np.int32), np.zeros(nE, np.float32)
    assert ctx.L.l3d_rdd_affinity(ctx.h, iters, _p(oi), _p(oj), _p(ow), C.c_longlong(nE)) == nE
    ri, rj, rw, _ = ctx.rdd(num_ids, ei, ej, ew, iters)
    key = ri.astype(np.int64) * num_ids + rj
    t = np.searchsorted(key, rj.astype(np.int64) * num_ids + ri)
    assert np.array_equal(key[t], rj.astype(np.int64) * num_ids + ri)          # every entry has its transposed entry
    assert _same((oi, oj, ow), (ri, rj, np.minimum(rw, rw[t])))
    assert np.any(rw != rw[t])                                                  # the min is not vacuous


def test_rdd_affinity_short_capacity_writes_nothing(affinity_ctx):
    ctx, ei, _, _, _ = affinity_ctx
    nE = len(ei)
    oi, oj, ow = np.full(nE, -7, np.int32), np.full(nE, -7, np.int32), np.full(nE, -7.0, np.float32)
    assert ctx.L.l3d_rdd_affinity(ctx.h, 10, _p(oi), _p(oj), _p(ow), C.c_longlong(nE - 1)) == nE
    assert np.all(oi == -7) and np.all(oj == -7) and np.all(ow == -7.0)


def test_rdd_argument_errors(gpu_ctx, oracle):
    L, h = gpu_ctx.L, gpu_ctx.h
    n, ei, ej, ew = rm.BUILDERS["tiny"]()
    ei, ej, ew = ei.copy(), ej.copy(), ew.copy()
    oi, oj, ow = np.full(2, -7, np.int32), np.full(2, -7, np.int32), np.full(2, -7.0, np.float32)
    args = [_p(ei), _p(ej), _p(ew), 10, _p(oi), _p(oj), _p(ow), None]
    for bad_n in (0, -1):
        assert L.l3d_rdd(h, bad_n, C.c_longlong(2), *args) == -1
        assert b"l3d_rdd" in L.l3d_last_error(h)
    for k in (0, 1, 2, 4, 5, 6):                        # a null array with nnz > 0
        a = list(args)
        a[k] = None
        assert L.l3d_rdd(h, n, C.c_longlong(2), *a) == -1, k
    assert L.l3d_rdd(h, n, C.c_longlong(0), *args) == 0     # nothing to diffuse: nothing written
    assert np.all(oi == -7) and np.all(oj == -7) and np.all(ow == -7.0)
    assert L.l3d_rdd(h, n, C.c_longlong(2), *args) == 0     # and the context still works
    assert _same((oi, oj, ow), oracle_rdd("tiny", 10))
