"""l3d_affinity_edges (the candidate list in emission order) against l3d_affinity_matrix: without collinearity links the matrix is
unused() and getLocalID (line3D.cc:1982-2023) restated here in numpy over the candidate list; with links every accepted edge is one
of the candidates, in candidate order."""
import ctypes as C

import numpy as np
import pytest

from line3dpp_b200 import synth
from tests import util

pytestmark = pytest.mark.gpu

TWO_SIGA_SQR, MIN_AFFINITY = 200.0, 0.5


def _scored_context(sc):
    """a context with the scene matched and scored (l3d_score_sweep), ready for the affinity calls"""
    from line3dpp_b200 import capi
    V = sc.num_views
    RtKinv, Cw = synth.camera_blocks(sc)
    k = [2.5 / sc.K[v][0, 0] for v in range(V)]          # spatial regulariser of 2.5 px (View::getSpecificSpatialReg)
    descs = capi.make_view_descs(sc.cam_ids, [sc.width] * V, [sc.height] * V, [len(s) for s in sc.segs], RtKinv, Cw, Cw, k, sc.median_depth)
    pairs = synth.view_pairs(sc.neighbors, sc.cam_ids)
    ctx = capi.Context(0)
    ctx.set_views(descs, sc.segs)
    ctx.match_pairs(pairs, util.pair_F(sc, pairs))
    assert ctx.L.l3d_score_sweep(ctx.h, C.c_float(TWO_SIGA_SQR), C.c_float(.5), C.c_float(.75), C.c_float(.1)) == 0
    return ctx, float(np.median(sc.median_depth))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def affinity_edges(ctx, med):
    args = (ctx.h, C.c_float(TWO_SIGA_SQR), C.c_float(med), C.c_float(MIN_AFFINITY))
    n = ctx._chk(ctx.L.l3d_affinity_edges(*args, None, None, None, C.c_longlong(0)), "l3d_affinity_edges")
    gi, gj, w = np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros(n, np.float32)
    assert ctx.L.l3d_affinity_edges(*args, _p(gi), _p(gj), _p(w), C.c_longlong(n)) == n
    return gi, gj, w


def affinity_matrix(ctx, med):
    args = (ctx.h, C.c_float(TWO_SIGA_SQR), C.c_float(med), C.c_float(MIN_AFFINITY))
    nids = C.c_longlong(0)
    n = ctx._chk(ctx.L.l3d_affinity_matrix(*args, None, None, None, C.c_longlong(0), None, C.c_longlong(0), C.byref(nids)), "l3d_affinity_matrix")
    ei, ej, ew, l2g = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.float32), np.zeros(nids.value, np.int64)
    assert ctx.L.l3d_affinity_matrix(*args, _p(ei), _p(ej), _p(ew), C.c_longlong(n), _p(l2g), C.c_longlong(len(l2g)), C.byref(nids)) == n
    return ei, ej, ew, l2g


@pytest.fixture(scope="module")
def plain():
    ctx, med = _scored_context(synth.make_scene(14, 500, 31, "ring3"))
    yield ctx, med
    ctx.close()


@pytest.fixture(scope="module")
def linked():
    ctx, med = _scored_context(synth.make_scene(12, 500, 93, "ring3", collinear=True))
    yield ctx, med
    ctx.close()


def test_matrix_is_unused_and_local_ids_of_the_edges(plain):
    ctx, med = plain
    gi, gj, w = affinity_edges(ctx, med)
    assert len(gi) > 1000
    # unused(): the first candidate of every unordered segment pair, in emission order
    key = np.minimum(gi, gj) << 32 | np.maximum(gi, gj)
    _, first = np.unique(key, return_index=True)
    keep = np.sort(first)
    assert len(keep) < len(gi)                            # the list really has repeated pairs
    a, b, wk = gi[keep], gj[keep], w[keep]
    # getLocalID: ids in order of first appearance, the source of an edge before its target
    seq = np.stack([a, b], 1).reshape(-1)
    segs, at = np.unique(seq, return_index=True)
    l2g = segs[np.argsort(at)]
    id_of = dict(zip(l2g.tolist(), range(len(l2g))))
    ia, ib = np.array([id_of[s] for s in a.tolist()], np.int32), np.array([id_of[s] for s in b.tolist()], np.int32)
    ei, ej, ew, m_l2g = affinity_matrix(ctx, med)
    assert np.array_equal(m_l2g, l2g)
    assert np.array_equal(ei, np.stack([ia, ib], 1).reshape(-1)) and np.array_equal(ej, np.stack([ib, ia], 1).reshape(-1))
    assert np.array_equal(util.bits(ew), util.bits(np.repeat(wk, 2)))


def test_linked_matrix_edges_are_candidates_in_order(linked):
    ctx, med = linked
    ctx.find_collinear(0.0, 0)
    n_plain = len(affinity_edges(ctx, med)[0])
    assert ctx.find_collinear(2.0, 0) > 1000
    gi, gj, w = affinity_edges(ctx, med)
    assert len(gi) > n_plain
    ei, ej, ew, l2g = affinity_matrix(ctx, med)
    assert len(ei) > 0
    # every accepted edge is a candidate with the same weight, and they come in candidate order: a subsequence of the list
    pos = 0
    for a, b, x in zip(l2g[ei[0::2]].tolist(), l2g[ej[0::2]].tolist(), util.bits(ew[0::2]).tolist()):
        hit = np.flatnonzero((gi[pos:] == a) & (gj[pos:] == b) & (util.bits(w[pos:]) == x))
        assert len(hit), (a, b)
        pos += int(hit[0]) + 1
