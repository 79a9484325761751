"""Line3D on a device list (matchImages splits the view pairs over several contexts and gathers the rows on the first) and the C ABI
call behind it, l3d_match_gather.  Every case compares with one device byte for byte.  On a single H100 the device lists repeat
device 0, which runs the same code path with device-to-device copies; [0, 1] runs when two GPUs are present."""
import ctypes as C

import numpy as np
import pytest

from line3dpp_b200 import capi, line3d, synth

pytestmark = pytest.mark.gpu

L3D_ERR_INVALID, L3D_ERR_STATE = -1, -3


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


def _run(scene, devices=None, knn=10, use_gpu=True, diffusion=False, collinearity=-1.0):
    kw = {} if devices is None else {"devices": devices}
    L = line3d.Line3D(neighbors_by_worldpoints=False, use_gpu=use_gpu, **kw)
    L.add_scene(scene)
    L.match_images(knn=knn)
    L.reconstruct_3d_lines(3, diffusion, collinearity)
    out, st = _dump(L, scene), L.stats()
    L.close()
    return out, st


def _check(scene, devices, **kw):
    want, ws = _run(scene, None, **kw)
    got, gs = _run(scene, devices, **kw)
    _same(got, want)
    assert gs["pair_evaluations"] == ws["pair_evaluations"] and gs["matches_after_knn"] == ws["matches_after_knn"]
    assert gs["lines3D"] == ws["lines3D"] > 0
    assert ws["ms_gather"] == 0.0 and gs["ms_gather"] >= 0.0


@pytest.fixture(scope="module")
def scene():
    return synth.make_scene(12, 400, 9, "ring3")


@pytest.mark.parametrize("knn", [10, -1, 40])
@pytest.mark.parametrize("devices", [[0, 0], [0, 0, 0]])
def test_device_list_equals_one_device(scene, devices, knn):
    _check(scene, devices, knn=knn)


@pytest.mark.parametrize("knn", [10, -1])
def test_device_list_ref_cpu_semantics(scene, knn):
    _check(scene, [0, 0], knn=knn, use_gpu=False)


def test_device_list_with_diffusion_and_collinearity(scene):
    _check(scene, [0, 0, 0], diffusion=True, collinearity=2.0)


def test_device_list_views_of_different_sizes():
    sc = synth.make_scene(12, 400, 21, "ring3")
    rng = np.random.default_rng(3)
    sc.segs = [s[:int(rng.integers(60, len(s) + 1))].copy() for s in sc.segs]
    assert len({len(s) for s in sc.segs}) > 6
    for knn in (10, -1):
        _check(sc, [0, 0, 0], knn=knn)


def test_more_devices_than_pairs():
    sc = synth.make_scene(4, 300, 5, "ring1")         # 4 view pairs over 6 contexts: some get none
    for knn in (10, -1):
        want, ws = _run(sc, None, knn=knn)
        got, gs = _run(sc, [0] * 6, knn=knn)
        _same(got, want)
        assert gs["pair_evaluations"] == ws["pair_evaluations"] and gs["matches_after_knn"] == ws["matches_after_knn"]


def test_two_gpus_equal_one(scene):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    for knn in (10, -1):
        _check(scene, [0, 1], knn=knn)


def test_bad_device_in_the_list_raises():
    with pytest.raises(capi.L3DError):
        line3d.Line3D(neighbors_by_worldpoints=False, devices=[0, 4096])
    with pytest.raises(capi.L3DError):
        line3d.Line3D(neighbors_by_worldpoints=False, devices=[-1])
    with pytest.raises(ValueError):
        line3d.Line3D(neighbors_by_worldpoints=False, devices=[])


# ---- the C ABI
def _job(sc):
    V = sc.num_views
    RtKinv, Cw = synth.camera_blocks(sc)
    k = [2.5 / sc.K[v][0, 0] for v in range(V)]
    descs = capi.make_view_descs(sc.cam_ids, [sc.width] * V, [sc.height] * V, [len(s) for s in sc.segs], RtKinv, Cw, Cw, k, sc.median_depth)
    pairs = synth.view_pairs(sc.neighbors, sc.cam_ids)
    Fd = np.stack([synth.fundamental(sc.K[s], sc.R[s], sc.t[s], sc.K[t], sc.R[t], sc.t[t]).reshape(9) for s, t in pairs])
    return descs, pairs, Fd


def _ctx(sc, descs):
    c = capi.Context(0)
    c.set_views(descs, sc.segs)
    return c


def _match(c, pairs, Fd, knn, first, last, f64=False):
    if f64:
        c.match_pairs_f64(pairs, Fd, 0.25, knn, first, last)
    else:
        c.match_pairs_range(pairs, Fd.astype(np.float32), first, last, 0.25, knn)


def _rows(c, sc, pairs):
    """every pair's counts and the records up to each row's count"""
    out = []
    for p, (s, _t) in enumerate(pairs):
        cnt, recs = c.pair_matches(p, len(sc.segs[s]))
        out.append((cnt.tobytes(), b"".join(recs[r, :cnt[r]].tobytes() for r in range(len(cnt)))))
    return out


def _figures(c):
    return (int(c.L.l3d_match_stride(c.h)), c.match_pair_evals(), int(c.L.l3d_match_total_matches(c.h)))


@pytest.fixture(scope="module")
def abi_scene():
    sc = synth.make_scene(10, 300, 13, "ring2")
    rng = np.random.default_rng(8)
    sc.segs = [s[:int(rng.integers(80, len(s) + 1))].copy() for s in sc.segs]
    return sc


@pytest.mark.parametrize("f64", [False, True])
@pytest.mark.parametrize("knn", [10, -1, 40])
def test_gather_equals_one_context(abi_scene, knn, f64):
    sc = abi_scene
    descs, pairs, Fd = _job(sc)
    n = len(pairs)
    one = _ctx(sc, descs)
    _match(one, pairs, Fd, knn, 0, n, f64)
    want, want_fig = _rows(one, sc, pairs), _figures(one)
    bounds = [0, 3, 3, n - 4, n]                       # one empty range
    srcs = [_ctx(sc, descs) for _ in range(4)]
    for i, s in enumerate(srcs):
        _match(s, pairs, Fd, knn, bounds[i], bounds[i + 1], f64)
    srcs[0].match_gather(srcs, bounds)                 # the destination is one of the sources
    srcs[0].sync()
    assert _rows(srcs[0], sc, pairs) == want and _figures(srcs[0]) == want_fig
    other = _ctx(sc, descs)                            # a destination that evaluated nothing itself
    _match(other, pairs, Fd, knn, 0, 0, f64)
    other.match_gather(srcs[1:], bounds[1:])
    sub = _ctx(sc, descs)
    _match(sub, pairs, Fd, knn, bounds[1], n, f64)
    assert _rows(other, sc, pairs) == _rows(sub, sc, pairs) and _figures(other) == _figures(sub)
    for c in srcs + [one, other, sub]:
        c.close()


def _sweep(c):
    return c.L.l3d_score_sweep(c.h, C.c_float(200.0), C.c_float(0.5), C.c_float(0.75), C.c_float(0.1))


def test_gather_rejects_other_jobs_and_bad_bounds(abi_scene):
    sc = abi_scene
    descs, pairs, Fd = _job(sc)
    n = len(pairs)
    h = n // 2
    a, b = _ctx(sc, descs), _ctx(sc, descs)

    def fresh(knn=10):
        _match(a, pairs, Fd, knn, 0, h)
        _match(b, pairs, Fd, knn, h, n)
        assert _sweep(a) == 0                          # a has a sweep, which every gather drops

    def rejected(code, srcs, bounds):
        rc = a.L.l3d_match_gather(a.h, len(srcs), (C.c_void_p * len(srcs))(*[s.h.value for s in srcs]),
                                  np.ascontiguousarray(bounds, np.int32).ctypes.data_as(C.c_void_p))
        assert rc == code, (rc, a.L.l3d_last_error(a.h))
        assert _sweep(a) == L3D_ERR_STATE              # no match result left
        assert a.L.l3d_match_stride(a.h) == L3D_ERR_STATE

    fresh()
    rejected(L3D_ERR_INVALID, [a, b], [0, h + 1, n])   # does not match what b evaluated
    fresh()
    rejected(L3D_ERR_INVALID, [a, b], [0, h, n + 1])   # outside the pair list
    fresh()
    rejected(L3D_ERR_INVALID, [b, a], [h, n, 0])       # decreasing
    fresh()
    _match(b, pairs, Fd * 1.5, 10, h, n)               # other matrices
    rejected(L3D_ERR_INVALID, [a, b], [0, h, n])
    fresh()
    _match(b, pairs[::-1].copy(), Fd[::-1].copy(), 10, h, n)      # another pair list
    rejected(L3D_ERR_INVALID, [a, b], [0, h, n])
    fresh()
    _match(b, pairs, Fd, 5, h, n)                      # another kNN
    rejected(L3D_ERR_INVALID, [a, b], [0, h, n])
    fresh()
    c = _ctx(sc, descs)                                # views, no match result
    rejected(L3D_ERR_STATE, [a, c], [0, h, n])
    fresh()
    b.set_views(descs, sc.segs)                        # a new upload drops b's match result
    rejected(L3D_ERR_STATE, [a, b], [0, h, n])
    # and the destination's own result must exist too
    fresh()
    a.set_views(descs, sc.segs)
    rejected(L3D_ERR_STATE, [a, b], [0, h, n])
    # success drops the sweep but keeps the gathered result; a sweep afterwards works
    fresh()
    a.match_gather([a, b], [0, h, n])
    assert _sweep(a) == 0
    for x in (a, b, c):
        x.close()
