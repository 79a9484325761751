"""Matching against caller-given candidates on the GPU (l3d_match_pairs_cand / _f64, k_match_cand; Line3D::setLineCandidates).

Every target as a candidate is the scan bit for bit; the candidates a plain run emitted (shuffled, duplicated, in both camera orders,
with random extras) give that run again; random subsets follow the model of tests/candidates_model.py row for row, while the scanned
pairs of the same call stay as they were; several devices and the lifecycle and error rules of the API."""
import ctypes as C

import numpy as np
import pytest

from line3dpp_b200 import capi, line3d, synth
from oracle import pyoracle
from tests import candidates_model as cm
from tests import util

pytestmark = pytest.mark.gpu

KNNS = [1, 10, 32, 0, 40]
PAIRS = [(0, 1), (1, 2), (2, 3), (3, 4), (4, 5), (5, 0), (1, 3)]
GEOMETRIES = ["sideways", "forward", "edge", "rolled"]


@pytest.fixture(scope="module")
def scene():
    return synth.make_scene(6, 400, 31, "ring2")


def _F(scene, pairs, f64):
    if not f64:
        return util.pair_F(scene, pairs)
    return np.stack([synth.fundamental(scene.K[s], scene.R[s], scene.t[s], scene.K[t], scene.R[t], scene.t[t]).reshape(9) for s, t in pairs])


def _result(ctx):
    row_ptr, recs = ctx.matches_csr()
    return dict(row_ptr=row_ptr, recs=recs.tobytes(), stride=int(ctx.L.l3d_match_stride(ctx.h)), total=int(ctx.L.l3d_match_total_matches(ctx.h)),
                evals=ctx.match_pair_evals())


def _plain(ctx, scene, pairs, knn, f64):
    F = _F(scene, pairs, f64)
    if f64:
        ctx.match_pairs_f64(pairs, F, 0.25, knn)
    else:
        ctx.match_pairs_range(pairs, F, 0, len(pairs), 0.25, knn)
    return _result(ctx)


def _cand(ctx, scene, pairs, knn, f64, restricted, triples, on_device=False):
    ctx.match_pairs_cand(pairs, _F(scene, pairs, f64), restricted, triples, 0.25, knn, f64=f64, on_device=on_device)
    return _result(ctx)


def _every_cell(scene, pairs, which):
    out = []
    for p in which:
        s, t = pairs[p]
        g = np.stack(np.meshgrid(np.arange(len(scene.segs[s])), np.arange(len(scene.segs[t])), indexing="ij"), -1).reshape(-1, 2)
        out.append(np.concatenate([np.full((len(g), 1), p), g], 1))
    return np.concatenate(out).astype(np.int32) if out else np.zeros((0, 3), np.int32)


def _same(a, b, evals=True):
    assert np.array_equal(a["row_ptr"], b["row_ptr"]) and a["recs"] == b["recs"] and a["stride"] == b["stride"] and a["total"] == b["total"]
    if evals:
        assert a["evals"] == b["evals"]


@pytest.mark.parametrize("f64", [False, True])
@pytest.mark.parametrize("knn", KNNS)
def test_every_target_is_the_scan(gpu_ctx, scene, f64, knn):
    """every pair restricted to all of its cells: counts, records, stride, total and evaluations bit-identical to the scan; every flag 0
    (with triples that are then ignored): the plain call byte for byte"""
    gpu_ctx.set_views(util.scene_descs(scene), scene.segs)
    pairs = np.array(PAIRS, np.int32)
    plain = _plain(gpu_ctx, scene, pairs, knn, f64)
    assert plain["total"] > 1000
    trip = _every_cell(scene, pairs, range(len(pairs)))
    _same(_cand(gpu_ctx, scene, pairs, knn, f64, np.ones(len(pairs)), trip), plain)
    _same(_cand(gpu_ctx, scene, pairs, knn, f64, np.zeros(len(pairs)), trip[::7]), plain)


@pytest.mark.parametrize("kind", GEOMETRIES)
@pytest.mark.parametrize("f64", [False, True])
@pytest.mark.parametrize("knn", [10, 0])
def test_every_target_special_geometry(gpu_ctx, kind, f64, knn):
    """the same on two-view scenes whose epipole lies inside, at the border of, outside or at infinity of the image"""
    sc = util.two_view_scene(kind, 500, 7)
    gpu_ctx.set_views(util.scene_descs(sc), sc.segs)
    pairs = np.array([(0, 1), (1, 0)], np.int32)
    plain = _plain(gpu_ctx, sc, pairs, knn, f64)
    assert plain["total"] > 100
    _same(_cand(gpu_ctx, sc, pairs, knn, f64, [1, 1], _every_cell(sc, pairs, [0, 1])), plain)


def test_every_target_epipole_vs_reference(gpu_ctx, ref_nofma):
    """epipole inside the image, every target listed: the verbatim reference wrapper's kNN rows (tests/test_match_gpu.py's rule)"""
    sc = util.two_view_scene("forward", 500, 7)
    gpu_ctx.set_views(util.scene_descs(sc), sc.segs)
    pairs = np.array([(0, 1)], np.int32)
    _cand(gpu_ctx, sc, pairs, 10, False, [1], _every_cell(sc, pairs, [0]))
    counts, recs = gpu_ctx.pair_matches(0, len(sc.segs[0]))
    pi = util.pair_inputs(sc, 0, 1)
    rc, ro, _, _ = pyoracle.match_lines(ref_nofma.ref_match_lines, pi["ls"], pi["lt"], pi["F"], pi["Rs"], pi["Rt"], pi["Cs"], pi["Ct"], 0, 1, 0.25, 10)
    assert np.array_equal(counts, rc) and counts.sum() > 100
    mine = util.rows_as_sets(counts, recs, ("tgt_seg", "overlap"))
    ref = util.rows_as_sets(rc, ro, ("tgt_seg", "overlap"))
    ties = sum(a != b for a, b in zip(mine, ref))
    assert ties <= 2


def _pair_rows(res, pairs, scene):
    """per pair: the (row_ptr slice, records) of the CSR result"""
    recs = np.frombuffer(res["recs"], capi.REC_DT)
    out, r0 = [], 0
    for s, _ in pairs:
        r1 = r0 + len(scene.segs[s])
        rp = res["row_ptr"][r0:r1 + 1]
        out.append((np.diff(rp).astype(np.int32), recs[rp[0]:rp[-1]]))
        r0 = r1
    return out


@pytest.mark.parametrize("f64", [False, True])
@pytest.mark.parametrize("knn", [10, 0, 40])
def test_random_subsets_follow_the_model(gpu_ctx, scene, f64, knn):
    """1 %, 10 % and 50 % of the cells of three pairs, an empty list on a fourth, the rest scanned: every restricted row is the model
    over the keep-all rows (records bit for bit), every scanned row is the plain call's; the evaluations count the distinct candidates"""
    gpu_ctx.set_views(util.scene_descs(scene), scene.segs)
    pairs = np.array(PAIRS, np.int32)
    rng = np.random.default_rng(knn + 100 * f64)
    keep_all = _pair_rows(_plain(gpu_ctx, scene, pairs, 0, f64), pairs, scene)
    plain = _pair_rows(_plain(gpu_ctx, scene, pairs, knn, f64), pairs, scene)
    restricted = np.zeros(len(pairs), np.int32)
    restricted[[0, 2, 4, 6]] = 1
    parts = []
    for p, frac in ((0, 0.01), (2, 0.10), (4, 0.50)):
        cells = _every_cell(scene, pairs, [p])
        pick = cells[rng.random(len(cells)) < frac]
        parts += [pick, pick[rng.integers(0, len(pick), len(pick) // 5)]]        # with duplicates
    parts.append(_every_cell(scene, pairs, [1])[::11])                          # a scanned pair's triples: ignored
    trip = np.concatenate(parts)
    trip = trip[rng.permutation(len(trip))]
    res = _cand(gpu_ctx, scene, pairs, knn, f64, restricted, trip)
    got = _pair_rows(res, pairs, scene)
    distinct = len({tuple(x) for x in trip.tolist() if restricted[x[0]]})
    scanned = sum(len(scene.segs[s]) * len(scene.segs[t]) for i, (s, t) in enumerate(pairs) if not restricted[i])
    assert res["evals"] == distinct + scanned
    for p in range(len(pairs)):
        counts, recs = got[p]
        if not restricted[p]:
            assert np.array_equal(counts, plain[p][0]) and recs.tobytes() == plain[p][1].tobytes(), p
            continue
        Ns = len(counts)
        ka_c, ka_r = keep_all[p]
        ka = np.zeros((Ns, max(1, int(ka_c.max()))), capi.REC_DT)
        off = np.concatenate([[0], np.cumsum(ka_c)])
        for r in range(Ns):
            ka[r, :ka_c[r]] = ka_r[off[r]:off[r + 1]]
        mine = trip[trip[:, 0] == p][:, 1:]
        mc, mm = cm.restricted_rows((ka_c, ka), mine, knn)
        assert np.array_equal(counts, mc), p
        exp = np.concatenate([mm[r, :mc[r]] for r in range(Ns)]) if mc.sum() else np.zeros(0, capi.REC_DT)
        assert recs.tobytes() == exp.tobytes(), p
        if p == 6:
            assert counts.sum() == 0
    assert sum(got[p][0].sum() for p in (0, 2, 4)) > 50


def test_random_subset_index_exact_to_the_oracle_model(gpu_ctx, scene):
    """the same restriction over the CPU oracle's keep-all rows (pyoracle.match_lines, knn = 0): the same target indices and overlap bits"""
    gpu_ctx.set_views(util.scene_descs(scene), scene.segs)
    pairs = np.array(PAIRS[:2], np.int32)
    rng = np.random.default_rng(3)
    cells = _every_cell(scene, pairs, [0])
    trip = cells[rng.random(len(cells)) < 0.1]
    for knn in (10, 0):
        got = _pair_rows(_cand(gpu_ctx, scene, pairs, knn, False, [1, 0], trip), pairs, scene)[0]
        mc, mm = cm.restricted_rows(cm.pair_keep_all(scene, 0, 1, 0.25, False), trip[:, 1:], knn)
        assert np.array_equal(got[0], mc) and mc.sum() > 20
        exp = np.concatenate([mm[r, :mc[r]] for r in range(len(mc))])
        assert np.array_equal(got[1]["tgt_seg"], exp["tgt_seg"]) and np.array_equal(util.bits(got[1]["overlap"]), util.bits(exp["overlap"]))


def test_on_device_triples(gpu_ctx, scene):
    """triples in device memory give the host-mode result"""
    import torch
    gpu_ctx.set_views(util.scene_descs(scene), scene.segs)
    pairs = np.array(PAIRS, np.int32)
    trip = _every_cell(scene, pairs, [1, 3])[::3]
    host = _cand(gpu_ctx, scene, pairs, 10, False, [0, 1, 0, 1, 0, 0, 0], trip)
    dev = torch.from_numpy(trip).cuda()
    torch.cuda.synchronize()
    _same(_cand(gpu_ctx, scene, pairs, 10, False, [0, 1, 0, 1, 0, 0, 0], (dev.data_ptr(), len(trip)), on_device=True), host)
    # filled by work queued on the context's stream just before the call, without a host synchronisation: the call reads them after it
    src = torch.from_numpy(trip).cuda()
    dev = torch.full_like(src, -1)
    torch.cuda.synchronize()
    with torch.cuda.stream(torch.cuda.ExternalStream(gpu_ctx.stream)):
        big = torch.empty(1 << 26, device="cuda")
        big.fill_(1.0)                                              # keeps the stream busy for a while first
        dev.copy_(src)
    _same(_cand(gpu_ctx, scene, pairs, 10, False, [0, 1, 0, 1, 0, 0, 0], (dev.data_ptr(), len(trip)), on_device=True), host)
    torch.cuda.synchronize()


def test_abi_errors(gpu_ctx, scene):
    gpu_ctx.set_views(util.scene_descs(scene), scene.segs)
    pairs = np.array(PAIRS[:2], np.int32)
    Ns, Nt = len(scene.segs[0]), len(scene.segs[1])
    for trip, msg in (([[2, 0, 0]], "outside the pair list"), ([[-1, 0, 0]], "outside the pair list"), ([[0, Ns, 0]], "outside the views"),
                      ([[0, 0, Nt]], "outside the views"), ([[1, -1, 0]], "outside the views")):
        launches = gpu_ctx.launch_count()
        with pytest.raises(capi.L3DError, match=msg):
            _cand(gpu_ctx, scene, pairs, 10, False, [1, 1], np.array(trip, np.int32))
        assert gpu_ctx.launch_count() == launches                 # rejected before anything is launched
        with pytest.raises(capi.L3DError, match="no match result"):
            gpu_ctx.match_counts()                                 # the failure dropped the match result
    F = util.pair_F(scene, pairs)
    rc = gpu_ctx.L.l3d_match_pairs_cand(gpu_ctx.h, 2, pairs.ctypes.data, F.ctypes.data, C.c_float(0.25), 10, 0, 2, None)
    assert rc == -1                                               # L3D_ERR_INVALID
    assert "null candidate descriptor" in gpu_ctx.L.l3d_last_error(gpu_ctx.h).decode()
    d = capi.CandDesc(None, None, 0, 0)
    assert gpu_ctx.L.l3d_match_pairs_cand(gpu_ctx.h, 2, pairs.ctypes.data, F.ctypes.data, C.c_float(0.25), 10, 0, 2, C.byref(d)) == -1
    d = capi.CandDesc(np.ones(2, np.int32).ctypes.data, None, 3, 0)
    assert gpu_ctx.L.l3d_match_pairs_cand(gpu_ctx.h, 2, pairs.ctypes.data, F.ctypes.data, C.c_float(0.25), 10, 0, 2, C.byref(d)) == -1
    # a restricted pair has no level-1 table or row windows; a scanned pair of the same call has them
    _cand(gpu_ctx, scene, pairs, 10, False, [1, 0], np.array([[0, 0, 0]], np.int32))
    with pytest.raises(capi.L3DError, match="restricted to caller-given candidates"):
        gpu_ctx.row_windows(0, Ns, Nt)
    win, _, off, _ = gpu_ctx.row_windows(1, len(scene.segs[1]), len(scene.segs[2]))
    assert off[-1] == len(scene.segs[2])


# ---- Line3D
def _line3d(sc, use_gpu=True, knn=10, lists=None, devices=None):
    L = line3d.Line3D(neighbors_by_worldpoints=False, use_gpu=use_gpu, devices=devices)
    L.add_scene(sc)
    for (a, b), v in (lists or {}).items():
        L.set_line_candidates(a, b, v)
    L.match_images(knn=knn)
    L.reconstruct_3d_lines(3, False)
    return L


def _outcome(L, sc):
    out = {f"scored_{c}": L.view_matches(c, False).tobytes() for c in sc.cam_ids}
    best, p = L.estimates()
    out["est"] = best.tobytes() + p.tobytes()
    out["aff"] = b"".join(np.ascontiguousarray(x).tobytes() for x in L.affinity())
    out["l2g"] = np.ascontiguousarray(L.local2global()).tobytes()
    out["seg3d"] = L.segments3d().tobytes()
    out["res"] = L.residuals().tobytes()
    out["lines"] = L.stats()["lines3D"]
    return out


def _emitted(L, sc):
    """{(src cam, tgt cam): [n, 2] emitted matches} of a Line3D's match result"""
    lib, h = capi.lib(), L.ctx
    pairs = L.pairs()
    off = np.zeros(len(pairs) + 1, np.int64)
    assert lib.l3d_pair_row_offsets(h, off.ctypes.data) == 0
    rows = int(off[-1])
    rp = np.zeros(rows + 1, np.int64)
    n = lib.l3d_get_matches_csr(h, rp.ctypes.data, None, 0)
    recs = np.zeros(max(n, 1), capi.REC_DT)
    lib.l3d_get_matches_csr(h, rp.ctypes.data, recs.ctypes.data, n)
    out = {}
    for p, (a, b) in enumerate(pairs):
        src = np.repeat(np.arange(off[p + 1] - off[p]), np.diff(rp[off[p]:off[p + 1] + 1]))
        out[(int(a), int(b))] = np.stack([src, recs[rp[off[p]]:rp[off[p + 1]]]["tgt_seg"].astype(np.int64)], 1)
    return out


@pytest.mark.parametrize("use_gpu", [True, False])
@pytest.mark.parametrize("knn", [10, 0])
def test_line3d_full_lists_and_emitted_lists(use_gpu, knn):
    """every cell listed, and then only the matches a plain run emitted (shuffled, duplicated, half the pairs in the other camera order,
    plus random extras): the plain run's scored matches, estimates, affinity, clusters and 3D lines"""
    sc = synth.make_scene(6, 250, 13, "ring2")
    L0 = _line3d(sc, use_gpu, knn)
    plain = _outcome(L0, sc)
    assert plain["lines"] > 10
    seg = {int(c): len(s) for c, s in zip(sc.cam_ids, sc.segs)}
    full = {(int(a), int(b)): np.stack(np.meshgrid(np.arange(seg[int(a)]), np.arange(seg[int(b)]), indexing="ij"), -1).reshape(-1, 2)
            for a, b in L0.pairs()}
    assert _outcome(_line3d(sc, use_gpu, knn, full), sc) == plain
    rng = np.random.default_rng(5)
    lists = {}
    for i, ((a, b), m) in enumerate(_emitted(L0, sc).items()):
        extra = np.stack([rng.integers(0, seg[a], 40), rng.integers(0, seg[b], 40)], 1)
        v = np.concatenate([m, m[: len(m) // 3], extra])
        v = v[rng.permutation(len(v))]
        lists[(b, a) if i % 2 else (a, b)] = v[:, ::-1] if i % 2 else v
    L1 = _line3d(sc, use_gpu, knn, lists)
    assert _outcome(L1, sc) == plain
    assert L1.stats()["pair_evaluations"] < L0.stats()["pair_evaluations"]


def test_line3d_subsets_vs_oracle_pipeline(ref_nofma):
    """10 % of the cells of two pairs, an empty list on a third: the product against OraclePipeline(match_source=model) over the verbatim
    reference kernels (the model's keep-all rows from its matcher, its scoring): scored matches (ids, overlaps, depths, score3D) bit for
    bit per view, and the number of 3D lines"""
    sc = synth.make_scene(6, 250, 17, "ring2")
    L0 = _line3d(sc)
    rng = np.random.default_rng(11)
    seg = {int(c): len(s) for c, s in zip(sc.cam_ids, sc.segs)}
    lists = {}
    for i, (a, b) in enumerate(L0.pairs()[:3]):
        a, b = int(a), int(b)
        cells = np.stack(np.meshgrid(np.arange(seg[a]), np.arange(seg[b]), indexing="ij"), -1).reshape(-1, 2)
        lists[(a, b)] = cells[rng.random(len(cells)) < 0.1] if i < 2 else np.zeros((0, 2), np.int64)
    L = _line3d(sc, lists=lists)
    O = pyoracle.OraclePipeline(False, True, match_source=cm.match_source(sc, lists, fn=ref_nofma.ref_match_lines), backend=ref_nofma)
    O.add_scene(sc)
    O.match_images()
    O.reconstruct(3, False)
    n = 0
    for cam in sc.cam_ids:
        a, b = L.view_matches(cam, False), O.scored(cam)
        assert len(a) == len(b) and np.array_equal(a["tgt_seg"], b["tgt_seg"]) and np.array_equal(a["tgt_cam"], b["tgt_cam"])
        for f in ("overlap", "score3D", "d_p1", "d_p2", "d_q1", "d_q2"):
            assert np.array_equal(util.bits(a[f]), util.bits(b[f])), (cam, f)
        n += len(a)
    assert n > 500
    assert abs(L.stats()["lines3D"] - O.num_lines()) <= max(2, O.num_lines() // 50)
    assert _outcome(L, sc) != _outcome(L0, sc)


def test_line3d_two_devices():
    """devices [0, 0]: the one-device result byte for byte"""
    sc = synth.make_scene(6, 250, 19, "ring2")
    rng = np.random.default_rng(2)
    pairs = _line3d(sc).pairs()
    seg = {int(c): len(s) for c, s in zip(sc.cam_ids, sc.segs)}
    lists = {(int(b), int(a)): np.stack([rng.integers(0, seg[int(b)], 3000), rng.integers(0, seg[int(a)], 3000)], 1) for a, b in pairs[::2]}
    for knn in (10, 0):
        one = _line3d(sc, knn=knn, lists=lists)
        two = _line3d(sc, knn=knn, lists=lists, devices=[0, 0])
        assert _outcome(one, sc) == _outcome(two, sc)
        assert one.stats()["pair_evaluations"] == two.stats()["pair_evaluations"]


def test_line3d_lifecycle_and_errors():
    sc = synth.make_scene(6, 250, 23, "ring2")
    L = _line3d(sc)
    plain = _outcome(L, sc)
    pairs = [tuple(int(x) for x in p) for p in L.pairs()]
    a, b = pairs[0]
    L.set_line_candidates(a, b, [[0, 0]])
    L.set_line_candidates(b, a, np.zeros((0, 2)))                  # replaces the list of the same pair
    L.match_images(); L.reconstruct_3d_lines(3, False)
    m = L.view_matches(a, False)
    assert not (m["tgt_cam"] == b).any()
    L.clear_line_candidates()                                      # every pair scanned again
    L.match_images(); L.reconstruct_3d_lines(3, False)
    assert _outcome(L, sc) == plain
    far = [(x, y) for x in sc.cam_ids for y in sc.cam_ids if x < y and (x, y) not in pairs and (y, x) not in pairs]
    assert far
    L.set_line_candidates(int(far[0][0]), int(far[0][1]), [[0, 0]])    # not visual neighbours: ignored
    L.set_line_candidates(12345, int(a), [[0, 0]])                 # a camera never added: ignored
    L.match_images(); L.reconstruct_3d_lines(3, False)
    assert _outcome(L, sc) == plain
    with pytest.raises(capi.L3DError, match="camA == camB"):
        L.set_line_candidates(a, a, [[0, 0]])
    assert L.L.l3dpp_set_line_candidates(L.h, a, b, None, 2) == -1                     # no array for two correspondences
    assert "no correspondence array" in L.L.l3dpp_last_error(L.h).decode()
    L.set_line_candidates(a, b, [[0, 0], [len(sc.segs[list(sc.cam_ids).index(a)]), 1]])
    with pytest.raises(capi.L3DError, match=f"segment {len(sc.segs[list(sc.cam_ids).index(a)])} of camera {a}"):
        L.match_images()
    assert L.stats()["view_pairs"] >= 0
    with pytest.raises(capi.L3DError):
        L.reconstruct_3d_lines(3, False)                           # no partial result: nothing to reconstruct from


@pytest.mark.parametrize("knn", [10, 0])
def test_setshard_with_lists_equals_unsharded(knn):
    """two emulated shards on one device (the in-process exchange of tests/test_dist_knn_gpu.py) with lopsided lists: small lists on the
    first half of the pairs and an empty one, so that the split weighted by listed correspondences differs from the Ns*Nt split.  Every
    rank ends with the unsharded result (same lists) byte for byte, and the evaluations of the ranks add up to the unsharded count."""
    import threading
    from tests.test_dist_knn_gpu import Exchange, _dump, _same
    sc = synth.make_scene(10, 300, 7, "ring3")
    seg = {int(c): len(s) for c, s in zip(sc.cam_ids, sc.segs)}
    probe = _line3d(sc)
    pairs = [(int(a), int(b)) for a, b in probe.pairs()]
    probe.close()
    rng = np.random.default_rng(9)
    lists, listed = {}, {}
    for i, (a, b) in enumerate(pairs[:len(pairs) // 2]):
        cells = np.stack(np.meshgrid(np.arange(seg[a]), np.arange(seg[b]), indexing="ij"), -1).reshape(-1, 2)
        v = np.zeros((0, 2), np.int64) if i == 1 else cells[rng.random(len(cells)) < 0.02]
        if i % 2:
            lists[(b, a)] = v[:, ::-1]                               # the other camera order
        else:
            lists[(a, b)] = v
        listed[(a, b)] = len(v)
    # the two splits of the pair list: by Ns*Nt, and as matchImages weighs it (a restricted pair by its listed correspondences)
    lib = capi.lib()
    ns_nt = np.array([seg[a] * seg[b] for a, b in pairs], np.int64)
    listed = np.array([listed.get((a, b), seg[a] * seg[b]) for a, b in pairs], np.int64)
    bounds = []
    for cost in (ns_nt, listed):
        bd = np.zeros(3, np.int32)
        assert lib.l3d_balanced_split(cost.ctypes.data, len(cost), 2, bd.ctypes.data) == 0
        bounds.append(bd)
    assert bounds[0][1] != bounds[1][1], bounds
    row_off = np.concatenate([[0], np.cumsum([seg[a] for a, _ in pairs])])

    full = _line3d(sc, knn=knn, lists=lists)
    full.reconstruct_3d_lines(3, True)
    want, want_st = _dump(full, sc), full.stats()
    full.close()

    ex, Ls, errs = Exchange(2), [], [None, None]
    for rank in range(2):
        L = line3d.Line3D(neighbors_by_worldpoints=False)
        L.add_scene(sc)
        for (a, b), v in lists.items():
            L.set_line_candidates(a, b, v)
        L._exchange_cb = ex.callback(rank)
        L._chk(L.L.l3dpp_set_shard(L.h, rank, 2, L._exchange_cb, None), "setShard")
        Ls.append(L)

    def run(rank):
        try:
            Ls[rank].match_images(knn=knn)
        except Exception as e:  # noqa: BLE001 - reported below
            errs[rank] = e
            ex.barrier.abort()
    th = [threading.Thread(target=run, args=(r,)) for r in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not ex.errors and errs == [None, None], (ex.errors, errs)
    try:
        rb = ex.calls[0][0][1]
        assert rb == [int(row_off[b]) for b in bounds[1]] and 0 < rb[1] < rb[2]      # the candidate-weighted bounds
        assert [k for k, _ in ex.calls[0]] == ([10] if knn == 10 else [0, int(Ls[0].L.l3d_match_stride(Ls[0].ctx))])
        assert sum(L.stats()["pair_evaluations"] for L in Ls) == want_st["pair_evaluations"]
        for L in Ls:
            L.reconstruct_3d_lines(3, True)
            _same(_dump(L, sc), want)
            assert L.stats()["lines3D"] == want_st["lines3D"] > 0
    finally:
        for L in Ls:
            L.close()
