"""Lens undistortion on the GPU (l3d_undistort_u8 / l3d_undistort_map / l3d_remap_u8, Line3D::undistortImage) against the numpy
restatement (tests/undistort_model.py) and what OpenCV computed (tests/golden/ref_undistort_v1.npz)."""
import ctypes as C

import numpy as np
import pytest

from line3dpp_b200 import capi, synth
from tests import undistort_model as um
from tests import util

pytestmark = pytest.mark.gpu

GOLDEN = um.__file__.replace("undistort_model.py", "golden/ref_undistort_v1.npz")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLDEN)


def _cases():
    return [str(n) for n in np.load(GOLDEN)["cases"]]


def _case(g, name):
    """(image, K, radial, tangential) of a golden case"""
    w, h, c, K, rad, tan = um.case_params(g, name)
    return um.make_image(h, w, c, seed=_cases().index(name)), K, rad, tan


@pytest.mark.parametrize("name", _cases())
def test_map_is_bit_identical_to_the_model(gpu_ctx, gold, name):
    img, K, rad, tan = _case(gold, name)
    h, w = img.shape[:2]
    xy, fr = gpu_ctx.undistort_map(w, h, K, rad, tan)
    mxy, mfr = um.model_maps_for(w, h, K, rad, tan)
    assert np.array_equal(xy, mxy) and np.array_equal(fr, mfr)


@pytest.mark.parametrize("name", _cases())
def test_remap_on_opencvs_maps_is_bit_exact(gpu_ctx, gold, name):
    """fed cv2's own maps (the model's plus the stored differing entries), l3d_remap_u8 reproduces cv2.remap byte for byte"""
    img, K, rad, tan = _case(gold, name)
    h, w = img.shape[:2]
    xy, fr = um.apply_corrections(*um.model_maps_for(w, h, K, rad, tan), gold[f"{name}/diff_idx"], gold[f"{name}/diff_xy"], gold[f"{name}/diff_frac"])
    assert um.sha(gpu_ctx.remap(img, xy, fr)) == str(gold[f"{name}/cv_remap_sha"])


def test_one_batched_call_over_every_case(gpu_ctx, gold):
    """one l3d_undistort_u8 launch over images of different sizes, channel counts and cameras, with row pitches above
    width * channels, on device memory; every output is what cv2.remap makes of the model's map.  Host mode gives the same bytes."""
    import torch
    names = _cases()
    cases = [_case(gold, n) for n in names]
    descs = (capi.UndistortDesc * len(cases))()
    srcs, dsts = [], []
    for i, (img, K, rad, tan) in enumerate(cases):
        h, w = img.shape[:2]
        c = 1 if img.ndim == 2 else 3
        sp, dp = w * c + 64 + 3 * i, w * c + 128 + i       # odd pitches: rows start at any byte
        s = torch.zeros((h, sp), dtype=torch.uint8, device="cuda")
        s[:, :w * c] = torch.from_numpy(img.reshape(h, w * c)).cuda()
        d = torch.full((h, dp), 77, dtype=torch.uint8, device="cuda")
        srcs.append(s); dsts.append(d)
        descs[i] = capi.make_undistort_desc(w, h, c, K, rad, tan, s.data_ptr(), sp, d.data_ptr(), dp)
    before = gpu_ctx.launch_count()
    gpu_ctx.undistort_device(descs)
    gpu_ctx.sync()
    assert gpu_ctx.launch_count() == before + 1
    dev = []
    for i, (name, (img, K, rad, tan)) in enumerate(zip(names, cases)):
        h, w = img.shape[:2]
        c = 1 if img.ndim == 2 else 3
        o = dsts[i].cpu().numpy()
        assert (o[:, w * c:] == 77).all(), "bytes beyond the row were written"
        out = np.ascontiguousarray(o[:, :w * c]).reshape(img.shape)
        assert um.sha(out) == str(gold[f"{name}/model_remap_sha"]), name
        dev.append(out)
    # host mode, inputs and outputs as row-padded views of wider arrays
    ins, outs = [], []
    for img, K, rad, tan in cases:
        wide = np.zeros((img.shape[0], img.shape[1] + 5) + img.shape[2:], np.uint8)
        wide[:, :img.shape[1]] = img
        ins.append(wide[:, :img.shape[1]])
        outs.append(np.zeros((img.shape[0], img.shape[1] + 9) + img.shape[2:], np.uint8)[:, :img.shape[1]])
    host = gpu_ctx.undistort(ins, [k for _, k, _, _ in cases], [r for _, _, r, _ in cases], [t for _, _, _, t in cases], out=outs)
    for a, b in zip(host, dev):
        assert np.array_equal(a, b)


def test_cpp_static_method_equals_the_c_abi(gpu_ctx, gold):
    """Line3D::undistortImage (through l3dpp_undistort_image) gives the bytes of l3d_undistort_u8; K's skew is ignored"""
    L = gpu_ctx.L
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    for name in ("colmap_opencv", "tiny", "vsfm"):
        img, K, rad, tan = _case(gold, name)
        h, w = img.shape[:2]
        c = 1 if img.ndim == 2 else 3
        out = np.zeros_like(img)
        K = np.ascontiguousarray(K, np.float64)
        assert L.l3dpp_undistort_image(p(img), p(out), h, w, c, p(np.array(rad, np.float64)), p(np.array(tan, np.float64)), p(K)) == 0
        assert np.array_equal(out, gpu_ctx.undistort([img], K, rad, tan)[0])
    img = um.make_image(5, 6, 1)
    bad = np.array([[0.0, 0, 3], [0, 10, 2], [0, 0, 1]])
    assert L.l3dpp_undistort_image(p(img), p(np.zeros_like(img)), 5, 6, 1, p(np.zeros(3)), p(np.zeros(2)), p(bad)) == -1


@pytest.mark.parametrize("shape", [(1, 1), (13, 17, 3), (480, 640), (257, 129, 3)])
def test_zero_distortion_is_the_identity(gpu_ctx, shape):
    img = um.make_image(shape[0], shape[1], 1 if len(shape) == 2 else 3, seed=5)
    K = np.array([[0.9 * shape[1] + 1, 0, shape[1] / 2 - 0.25], [0, 0.8 * shape[0] + 1, shape[0] / 2 + 0.375], [0, 0, 1]])
    assert np.array_equal(gpu_ctx.undistort([img], K)[0], img)


def _reject_cases():
    ok = dict(width=64, height=48, channels=1, K=np.array([[50.0, 0, 32], [0, 50, 24], [0, 0, 1]]), radial=(0.1, 0, 0), tangential=(0, 0))
    bad = []
    for k, v in (("width", 0), ("width", 32768), ("height", 0), ("height", 40000), ("channels", 2), ("channels", 4)):
        bad.append((f"{k}={v}", dict(ok, **{k: v}), None))
    for key, val in (("fx", 0.0), ("fy", 0.0), ("fx", np.inf), ("fy", np.nan), ("cx", np.nan)):
        K = ok["K"].copy()
        K[{"fx": (0, 0), "fy": (1, 1), "cx": (0, 2)}[key]] = val
        bad.append((f"{key}={val}", dict(ok, K=K), None))
    bad.append(("k3=inf", dict(ok, radial=(0.1, 0, np.inf)), None))
    bad.append(("p2=nan", dict(ok, tangential=(0, np.nan)), None))
    bad += [("src_pitch", ok, "src_pitch"), ("dst_pitch", ok, "dst_pitch"), ("null src", ok, "src"), ("null dst", ok, "dst"), ("src==dst", ok, "alias")]
    return bad


def test_rejected_arguments(gpu_ctx):
    """each bad argument returns L3D_ERR_INVALID from every call that uses it"""
    L = gpu_ctx.L
    src, dst = np.zeros(64 * 48 * 3, np.uint8), np.zeros(64 * 48 * 3, np.uint8)
    xy, fr = np.zeros(64 * 48 * 2, np.int16), np.zeros(64 * 48, np.uint16)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    for what, a, field in _reject_cases():
        d = capi.make_undistort_desc(a["width"], a["height"], a["channels"], a["K"], a["radial"], a["tangential"], src.ctypes.data, None,
                                     dst.ctypes.data, None)
        if field == "src_pitch":
            d.src_pitch = 63
        elif field == "dst_pitch":
            d.dst_pitch = 10
        elif field in ("src", "dst"):
            setattr(d, field, None)
        elif field == "alias":
            d.dst = d.src
        assert L.l3d_undistort_u8(gpu_ctx.h, 1, C.byref(d), 0) == -1, what
        image_arg = field is not None or what.split("=")[0] in ("width", "height", "channels")
        camera_arg = field is None
        if camera_arg:
            assert L.l3d_undistort_map(gpu_ctx.h, C.byref(d), p(xy), p(fr), 0) == -1, what
        if image_arg:
            assert L.l3d_remap_u8(gpu_ctx.h, C.byref(d), p(xy), p(fr), 0) == -1, what
    d = capi.make_undistort_desc(64, 48, 1, _reject_cases()[0][1]["K"], src=src.ctypes.data, dst=dst.ctypes.data)
    assert L.l3d_undistort_u8(gpu_ctx.h, -1, C.byref(d), 0) == -1
    assert L.l3d_undistort_u8(gpu_ctx.h, 1, None, 0) == -1
    assert L.l3d_undistort_map(gpu_ctx.h, C.byref(d), None, p(fr), 0) == -1
    assert L.l3d_remap_u8(gpu_ctx.h, C.byref(d), p(xy), None, 0) == -1
    assert L.l3d_undistort_u8(gpu_ctx.h, 1, C.byref(d), 0) == 0


def test_undistort_calls_leave_the_pipeline_results_alone(gold):
    """a context holding matches, a score sweep and an affinity matrix gives the same view matches and diffusion result after
    undistortion calls, successful and rejected"""
    sc = synth.make_scene(14, 500, 31, "ring3")
    V = sc.num_views
    RtKinv, Cw = synth.camera_blocks(sc)
    k = [2.5 / sc.K[v][0, 0] for v in range(V)]
    descs = capi.make_view_descs(sc.cam_ids, [sc.width] * V, [sc.height] * V, [len(s) for s in sc.segs], RtKinv, Cw, Cw, k, sc.median_depth)
    pairs = synth.view_pairs(sc.neighbors, sc.cam_ids)
    ctx = capi.Context(0)
    L = ctx.L
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    ctx.set_views(descs, sc.segs)
    ctx.match_pairs(pairs, util.pair_F(sc, pairs))
    assert L.l3d_score_sweep(ctx.h, C.c_float(200), C.c_float(.5), C.c_float(.75), C.c_float(.1)) == 0
    nids = C.c_longlong(0)
    nE = L.l3d_affinity_matrix(ctx.h, C.c_float(200), C.c_float(float(np.median(sc.median_depth))), C.c_float(.5), None, None, None,
                               C.c_longlong(0), None, C.c_longlong(0), C.byref(nids))
    assert nE > 0

    def results():
        views = []
        for v in range(V):
            n = L.l3d_get_view_matches(ctx.h, v, 0, None, C.c_longlong(0))
            m = np.zeros(max(n, 1), capi.MATCH_DT)
            assert L.l3d_get_view_matches(ctx.h, v, 0, p(m), C.c_longlong(len(m))) == n
            views.append(m[:n].tobytes())
        oi, oj, ow = np.zeros(nE, np.int32), np.zeros(nE, np.int32), np.zeros(nE, np.float32)
        n = L.l3d_rdd_affinity(ctx.h, 10, p(oi), p(oj), p(ow), C.c_longlong(nE))
        assert n > 0
        return views, oi[:n].tobytes() + oj[:n].tobytes() + ow[:n].tobytes()

    before = results()
    img, K, rad, tan = _case(gold, "colmap_opencv")
    ctx.undistort([img, img[:, :, 0].copy()], K, rad, tan)
    ctx.undistort_map(img.shape[1], img.shape[0], K, rad, tan)
    ctx.remap(img, *um.model_maps_for(img.shape[1], img.shape[0], K, rad, tan))
    for bad_K in (np.zeros((3, 3)), np.array([[1.0, 0, 0], [0, np.nan, 0], [0, 0, 1]])):
        with pytest.raises(capi.L3DError, match=r"failed \(-1\)"):
            ctx.undistort([img], bad_K)
        with pytest.raises(capi.L3DError, match=r"failed \(-1\)"):
            ctx.undistort_map(img.shape[1], img.shape[0], bad_K)
    with pytest.raises(capi.L3DError, match=r"failed \(-1\)"):
        ctx.undistort([np.zeros((0, 4), np.uint8)], K)                   # height 0
    assert results() == before
    ctx.close()
