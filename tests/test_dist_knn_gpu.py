"""Sharded matchImages in the keep-all (kNN <= 0) and kNN > 32 modes (Line3D::setShard): the exchange callback runs twice, first
for the row counts alone (knn = 0), then, after every rank has re-laid its records at the longest row of the whole job
(l3d_match_restride), for the rows at that stride.  Every rank must end with the unsharded result bit for bit.

The ranks run in one process on one device: one Line3D per rank, each matching on its own thread (ctypes releases the GIL), and an
in-process exchange that meets at a barrier and copies every row from its owner's buffer, which is what one broadcast per owner does
over NCCL.  Two real processes over NCCL run when the box has >= 2 GPUs."""
import collections
import ctypes as C
import os
import socket
import subprocess
import sys
import textwrap
import threading

import numpy as np
import pytest

from line3dpp_b200 import capi, line3d, synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REC = 24
L3D_ERR_INVALID, L3D_ERR_STATE = -1, -3


def crowded_scene(views, segs, seed, ring, crowd_views=3, copies=60):
    """a ring scene in which the first `crowd_views` views each hold `copies` extra copies of one 3D line's segment, offset by
    0.05 px steps across it: the rows of their pairs get about `copies` matches (the other rows a handful), so kNN = 40 cuts them
    and the ranks that match those pairs have a wider own stride than the rest"""
    sc = synth.make_scene(views, segs, seed, ring)
    seen = collections.Counter(int(l) for ids in sc.line_ids[:crowd_views] for l in set(ids.tolist()))
    line = min(seen, key=lambda l: (-seen[l], l))
    for v in range(crowd_views):
        hit = np.flatnonzero(sc.line_ids[v] == line)
        if len(hit) == 0:
            continue
        s = sc.segs[v][hit[0]].astype(np.float64)
        d = s[2:] - s[:2]
        n = np.array([-d[1], d[0]]) / np.linalg.norm(d)
        off = (np.arange(1, copies + 1) * 0.05)[:, None] * n[None, :]
        sc.segs[v] = np.concatenate([sc.segs[v], np.concatenate([s[:2] + off, s[2:] + off], axis=1).astype(np.float32)])
    return sc


@pytest.fixture(scope="module")
def scene():
    return crowded_scene(10, 300, 7, "ring3")


def _dump(L, scene):
    out = {"est": L.estimates(), "aff": L.affinity(raw=True), "seg3d": L.segments3d(), "resid": L.residuals()}
    out["kept"] = [L.view_matches(c, True) for c in scene.cam_ids]
    return out


def _same(a, b):
    assert a["est"][0].tobytes() == b["est"][0].tobytes() and a["est"][1].tobytes() == b["est"][1].tobytes()
    assert len(a["kept"]) == len(b["kept"])
    for x, y in zip(a["kept"], b["kept"]):
        assert x.tobytes() == y.tobytes()
    for x, y in zip(a["aff"], b["aff"]):
        assert x.tobytes() == y.tobytes()
    assert a["seg3d"].tobytes() == b["seg3d"].tobytes() and a["resid"].tobytes() == b["resid"].tobytes()


def _stride(L):
    return int(L.L.l3d_match_stride(L.ctx))


def _unsharded(scene, knn, use_gpu):
    L = line3d.Line3D(neighbors_by_worldpoints=False, use_gpu=use_gpu)
    L.add_scene(scene)
    L.match_images(knn=knn)
    stride = _stride(L)
    L.reconstruct_3d_lines(3, True)
    out, st = _dump(L, scene), L.stats()
    L.close()
    return out, st, stride


class Exchange:
    """the exchange of `world` ranks in one process: every rank publishes its buffers, waits for the others, copies the rows it does
    not own from their owners and waits again, so that no rank re-lays or frees its buffers while another still reads them"""

    def __init__(self, world):
        self.barrier = threading.Barrier(world, timeout=300)
        self.bufs = [None] * world
        self.calls = [[] for _ in range(world)]
        self.errors = []

    def callback(self, rank):
        import torch
        from line3dpp_b200 import dist as l3dist

        def cb(_user, counts_dev, recs_dev, row_bounds, world, knn):
            try:
                rb = [row_bounds[i] for i in range(world + 1)]
                self.calls[rank].append((knn, rb))
                counts = l3dist.device_bytes(counts_dev, 4 * rb[-1], 0)
                recs = l3dist.device_bytes(recs_dev, REC * knn * rb[-1], 0)
                torch.cuda.synchronize()
                self.bufs[rank] = (counts, recs, rb, knn)
                self.barrier.wait()
                for r in range(world):
                    a, b = rb[r], rb[r + 1]
                    if r == rank or b <= a:
                        continue
                    oc, orecs, orb, oknn = self.bufs[r]
                    assert orb == rb and oknn == knn, "the ranks disagree on the row bounds or the stride"
                    counts[4 * a:4 * b] = oc[4 * a:4 * b]
                    recs[REC * knn * a:REC * knn * b] = orecs[REC * knn * a:REC * knn * b]
                torch.cuda.synchronize()
                self.barrier.wait()
                return 0
            except Exception as e:  # noqa: BLE001 - must not unwind through the C frame
                self.errors.append(e)
                self.barrier.abort()
                return -1
        return l3dist._EXCHANGE_T(cb)


def _sharded(scene, knn, use_gpu, world, devices=None):
    """one Line3D per rank (rank r on devices[r] if given), matched concurrently; returns the Line3Ds, their strides and the exchange"""
    ex = Exchange(world)
    Ls = []
    for rank in range(world):
        kw = {} if devices is None or devices[rank] is None else {"devices": devices[rank]}
        L = line3d.Line3D(neighbors_by_worldpoints=False, use_gpu=use_gpu, **kw)
        L.add_scene(scene)
        L._exchange_cb = ex.callback(rank)
        L._chk(L.L.l3dpp_set_shard(L.h, rank, world, L._exchange_cb, None), "setShard")
        Ls.append(L)
    errs = [None] * world

    def run(rank):
        try:
            Ls[rank].match_images(knn=knn)
        except Exception as e:  # noqa: BLE001 - reported below
            errs[rank] = e
            ex.barrier.abort()
    th = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not ex.errors, ex.errors
    assert errs == [None] * world, errs
    return Ls, [_stride(L) for L in Ls], ex


def _check(scene, knn, use_gpu, world, devices=None):
    want, ws, want_stride = _unsharded(scene, knn, use_gpu)
    Ls, strides, ex = _sharded(scene, knn, use_gpu, world, devices)
    try:
        for rank, L in enumerate(Ls):
            calls = ex.calls[rank]
            assert [k for k, _ in calls] == [0, strides[rank]], calls      # the counts, then the rows at the common stride
            assert calls[0][1] == calls[1][1]
        assert len(set(strides)) == 1
        if knn <= 0:
            assert strides[0] == want_stride                               # the longest row of the whole job
        else:
            assert strides[0] <= min(knn, want_stride)                     # the longest row after the cut
        st = [L.stats() for L in Ls]
        assert sum(s["pair_evaluations"] for s in st) == ws["pair_evaluations"]
        for L, s in zip(Ls, st):
            assert s["matches_after_knn"] == ws["matches_after_knn"]
            L.reconstruct_3d_lines(3, True)
            _same(_dump(L, scene), want)
            assert L.stats()["lines3D"] == ws["lines3D"] > 0
    finally:
        for L in Ls:
            L.close()
    return ex, strides, want_stride


@pytest.mark.parametrize("use_gpu", [True, False])
@pytest.mark.parametrize("knn", [-1, 40])
@pytest.mark.parametrize("world", [2, 3])
def test_sharded_keep_all_and_wide_knn_equal_unsharded(scene, world, knn, use_gpu):
    ex, strides, want_stride = _check(scene, knn, use_gpu, world)
    rb = ex.calls[0][0][1]
    assert all(rb[r] < rb[r + 1] for r in range(world)), "every rank must own rows"
    if knn > 0:
        assert strides[0] == knn < want_stride        # the crowded rows are cut: the sharded stride is narrower than one context's


def test_more_ranks_than_view_pairs():
    sc = crowded_scene(4, 300, 5, "ring1", crowd_views=2)      # 4 view pairs over 6 ranks: some match nothing
    for knn in (-1, 40):
        ex, _, _ = _check(sc, knn, True, 6)
        rb = ex.calls[0][0][1]
        assert any(rb[r] == rb[r + 1] for r in range(6))


@pytest.mark.parametrize("knn", [-1, 40])
def test_device_list_inside_a_shard(scene, knn):
    _check(scene, knn, True, 2, devices=[[0, 0], None])


# ---- the exchange callback's failures
def test_failing_exchange_leaves_no_result(scene):
    from line3dpp_b200 import dist as l3dist
    L = line3d.Line3D(neighbors_by_worldpoints=False)
    L.add_scene(scene)
    calls, fail_at = [], [0]

    def cb(_u, _counts, _recs, row_bounds, world, knn):
        calls.append(knn)
        return -1 if len(calls) == fail_at[0] else 0     # no rows move: rank 1's share stays empty, which matchImages cannot tell
    fn = l3dist._EXCHANGE_T(cb)
    # top-k: one call with knn = kNN
    L._chk(L.L.l3dpp_set_shard(L.h, 0, 2, fn, None), "setShard")
    L.match_images(knn=10)
    assert calls == [10]
    for knn in (-1, 40):
        for fail_at[0] in (1, 2):
            L._chk(L.L.l3dpp_set_shard(L.h, 0, 1, None, None), "setShard")
            L.match_images(knn=knn)
            L.reconstruct_3d_lines(3, True)
            assert L.stats()["lines3D"] > 0 and len(L.estimates()[0]) > 0
            L._chk(L.L.l3dpp_set_shard(L.h, 0, 2, fn, None), "setShard")
            calls.clear()
            with pytest.raises(capi.L3DError, match="exchange callback failed"):
                L.match_images(knn=knn)
            assert "exchange callback failed" in L.L.l3dpp_last_error(L.h).decode()
            assert len(calls) == fail_at[0] and calls[0] == 0
            if fail_at[0] == 2:
                assert calls[1] == _stride(L) >= 1
            assert len(L.estimates()[0]) == 0                      # the earlier run's estimates are gone
            with pytest.raises(capi.L3DError, match="no clusterable segments"):
                L.reconstruct_3d_lines(3, True)
    L.close()


# ---- l3d_match_restride through the C ABI
def _job(sc):
    V = sc.num_views
    RtKinv, Cw = synth.camera_blocks(sc)
    k = [2.5 / sc.K[v][0, 0] for v in range(V)]
    descs = capi.make_view_descs(sc.cam_ids, [sc.width] * V, [sc.height] * V, [len(s) for s in sc.segs], RtKinv, Cw, Cw, k, sc.median_depth)
    pairs = synth.view_pairs(sc.neighbors, sc.cam_ids)
    F = np.stack([synth.fundamental(sc.K[s], sc.R[s], sc.t[s], sc.K[t], sc.R[t], sc.t[t]).reshape(9) for s, t in pairs]).astype(np.float32)
    return descs, pairs, F


def _rows(c, sc, pairs):
    """every pair's counts and the records up to each row's count"""
    out = []
    for p, (s, _t) in enumerate(pairs):
        cnt, recs = c.pair_matches(p, len(sc.segs[s]))
        out.append((cnt.tobytes(), b"".join(recs[r, :cnt[r]].tobytes() for r in range(len(cnt)))))
    return out


def _sweep(c):
    return c.L.l3d_score_sweep(c.h, C.c_float(200.0), C.c_float(0.5), C.c_float(0.75), C.c_float(0.1))


def _estimates(c):
    n = c.L.l3d_get_estimates(c.h, None, None, C.c_longlong(0))
    if n < 0:
        return n
    best, p = np.zeros(n, capi.MATCH_DT), np.zeros((n, 6), np.float64)
    c.L.l3d_get_estimates(c.h, best.ctypes.data_as(C.c_void_p), p.ctypes.data_as(C.c_void_p), C.c_longlong(n))
    return best.tobytes() + p.tobytes()


@pytest.mark.parametrize("knn", [-1, 40, 10])
def test_restride_wider_then_narrower_keeps_every_row(scene, knn):
    descs, pairs, F = _job(scene)
    c = capi.Context(0)
    c.set_views(descs, scene.segs)
    c.match_pairs(pairs, F, 0.25, knn)
    stride0 = c._knn
    counts, _ = c.match_counts()
    longest = max(int(counts.max()), 1)
    want = _rows(c, scene, pairs)
    assert _sweep(c) == 0
    want_est = _estimates(c)
    assert c.match_restride(stride0 + 17) == stride0 + 17 == c.L.l3d_match_stride(c.h)
    assert _estimates(c) == L3D_ERR_STATE                  # the sweep is dropped
    assert _rows(c, scene, pairs) == want
    assert _sweep(c) == 0 and _estimates(c) == want_est    # and the sweep at the new stride gives the same estimates
    assert c.match_restride(0) == longest == c.L.l3d_match_stride(c.h)
    assert _rows(c, scene, pairs) == want
    if knn == 40:
        assert longest == 40 < stride0                     # narrower than the stride matching chose (the longest row before the cut)
    assert c.match_restride(longest) == longest            # the same stride: nothing moves
    assert _rows(c, scene, pairs) == want
    c.close()


def test_restride_rejects_and_drops_the_result(scene):
    descs, pairs, F = _job(scene)
    c = capi.Context(0)
    c.set_views(descs, scene.segs)
    assert c.L.l3d_match_restride(c.h, 0) == L3D_ERR_STATE                 # views, no match result
    for bad in ("short", "huge"):
        c.match_pairs(pairs, F, 0.25, -1)
        assert _sweep(c) == 0
        rows = c.match_total_rows()
        stride = 39 if bad == "short" else (1 << 31) // rows + 1          # below the longest row (61), or 2^31 slots
        assert c.L.l3d_match_restride(c.h, stride) == L3D_ERR_INVALID, c.L.l3d_last_error(c.h)
        assert _sweep(c) == L3D_ERR_STATE                                  # no match result left
        assert c.L.l3d_match_stride(c.h) == L3D_ERR_STATE
        assert c.L.l3d_match_restride(c.h, 0) == L3D_ERR_STATE
    c.close()


# ---- two processes over NCCL
WORKER = textwrap.dedent("""
    import os, sys, numpy as np, torch, torch.distributed as dist
    sys.path.insert(0, %r)
    from line3dpp_b200 import line3d, synth, dist as l3dist
    from tests.test_dist_knn_gpu import crowded_scene
    dev = int(os.environ["LOCAL_RANK"]); torch.cuda.set_device(dev)
    dist.init_process_group("nccl", device_id=torch.device("cuda", dev))
    scene = crowded_scene(12, 400, 9, "ring3")
    def dump(L):
        b, p = L.estimates(); s, r = L.segments3d(), L.residuals()
        return b.tobytes() + p.tobytes() + s.tobytes() + r.tobytes() + b"".join(L.view_matches(c, True).tobytes() for c in scene.cam_ids)
    full = line3d.Line3D(neighbors_by_worldpoints=False, device=dev)
    full.add_scene(scene); full.match_images(knn=-1)
    stride = full.L.l3d_match_stride(full.ctx)
    full.reconstruct_3d_lines(3, True)
    L = line3d.Line3D(neighbors_by_worldpoints=False, device=dev)
    L.add_scene(scene)
    keep = l3dist.attach(L, dev)
    L.match_images(knn=-1)
    assert L.L.l3d_match_stride(L.ctx) == stride
    assert [c["knn"] for c in L._exchange_state["exchanges"]] == [0, stride]
    L.reconstruct_3d_lines(3, True)
    assert L.stats()["pair_evaluations"] < full.stats()["pair_evaluations"], "this rank evaluated every pair"
    assert L.stats()["lines3D"] == full.stats()["lines3D"] > 50
    assert L.stats()["matches_after_knn"] == full.stats()["matches_after_knn"]
    assert dump(L) == dump(full), "sharded result differs from the single-GPU result"
    dist.barrier(); L.close(); full.close(); dist.destroy_process_group()
    print("rank", dev, "sharded keep-all == unsharded")
""")


def test_two_process_nccl_keep_all_equals_single_gpu(tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    script = tmp_path / "worker.py"
    script.write_text(WORKER % ROOT)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), str(script)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, NCCL_DEBUG="WARN"))
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
