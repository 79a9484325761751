"""The rational and fisheye lens models of l3d_undistort.cu on the GPU against the restatement (tests/lens_model.py) and what OpenCV
computed (tests/golden/ref_undistort_lens_v1.npz); the pinhole cases of ref_undistort_v1.npz through the new descriptor fields."""
import ctypes as C
import os

import numpy as np
import pytest

from line3dpp_b200 import capi, line3d, synth
from tests import lens_model as lm
from tests import undistort_model as um
from tests import util

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "ref_undistort_lens_v1.npz")
PINHOLE_GOLDEN = os.path.join(HERE, "golden", "ref_undistort_v1.npz")
# the fisheye map may differ from cv2's where the device's atan and glibc's differ in the last ulp and that moves u or v across a
# rounding boundary: at most this many entries per million beyond the restatement's own difference count (DESIGN.md §4a)
FISHEYE_EXTRA_PER_MILLION = 20


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLDEN)


def _cases(model=None):
    g = np.load(GOLDEN)
    return [str(n) for n in g["cases"] if model is None or int(g[f"{n}/model"]) == model]


def _lens(model, k, p):
    return dict(model=int(model), k=np.asarray(k, np.float64), p=np.asarray(p, np.float64))


def _case(g, name):
    """(image, K, lens) of a golden case"""
    w, h, c, K, model, k, p = lm.case_params(g, name)
    return um.make_image(h, w, c, seed=100 + _cases().index(name)), K, _lens(model, k, p)


def _fixed(xy, fr):
    """(u, v) in 1/32 px of fixed-point maps"""
    return xy[..., 0].astype(np.int64) * 32 + (fr & 31), xy[..., 1].astype(np.int64) * 32 + (fr >> 5)


@pytest.mark.parametrize("name", _cases(lm.RADTAN))
def test_rational_map_is_bit_identical_to_the_model(gpu_ctx, gold, name):
    img, K, lens = _case(gold, name)
    h, w = img.shape[:2]
    xy, fr = gpu_ctx.undistort_map(w, h, K, lens=lens)
    mxy, mfr = lm.model_maps_for(w, h, K, lens["model"], lens["k"], lens["p"])
    assert np.array_equal(xy, mxy) and np.array_equal(fr, mfr)


@pytest.mark.parametrize("name", _cases(lm.FISHEYE))
def test_fisheye_map_is_within_one_step_of_opencv(gpu_ctx, gold, name):
    img, K, lens = _case(gold, name)
    h, w = img.shape[:2]
    xy, fr = gpu_ctx.undistort_map(w, h, K, lens=lens)
    mxy, mfr = lm.model_maps_for(w, h, K, lens["model"], lens["k"], lens["p"])
    cxy, cfr = um.apply_corrections(mxy, mfr, gold[f"{name}/diff_idx"], gold[f"{name}/diff_xy"], gold[f"{name}/diff_frac"])
    assert um.sha(cxy, cfr) == str(gold[f"{name}/cv_map_sha"])
    (gu, gv), (cu, cv) = _fixed(xy, fr), _fixed(cxy, cfr)
    du, dv = np.abs(gu - cu), np.abs(gv - cv)
    if name == "fisheye_int16":                 # wrapped entries: compare modulo the int16 range of the pixel part
        du, dv = np.minimum(du, 65536 * 32 - du), np.minimum(dv, 65536 * 32 - dv)
    assert du.max() <= 1 and dv.max() <= 1
    differ = int(((du != 0) | (dv != 0)).sum())
    model_differ = len(gold[f"{name}/diff_idx"])
    print(f"fisheye {name}: {differ} of {w * h} map entries differ from cv2's (restatement: {model_differ})")
    assert differ <= model_differ + FISHEYE_EXTRA_PER_MILLION * w * h // 1_000_000 + 1


@pytest.mark.parametrize("name", _cases())
def test_fused_output_is_the_remap_of_its_own_map(gpu_ctx, gold, name):
    img, K, lens = _case(gold, name)
    h, w = img.shape[:2]
    xy, fr = gpu_ctx.undistort_map(w, h, K, lens=lens)
    fused = gpu_ctx.undistort([img], K, lens=lens)[0]
    assert np.array_equal(fused, gpu_ctx.remap(img, xy, fr))
    if lens["model"] == lm.RADTAN:              # the rational map is the model's: cv2.remap of it is stored
        assert um.sha(fused) == str(gold[f"{name}/model_remap_sha"])


def test_pinhole_cases_through_the_new_fields_are_unchanged(gpu_ctx):
    """every case of ref_undistort_v1.npz with model = RADTAN and zero rational terms set explicitly gives today's bytes"""
    g = np.load(PINHOLE_GOLDEN)
    names = [str(n) for n in g["cases"]]
    for i, name in enumerate(names):
        w, h, c, K, rad, tan = um.case_params(g, name)
        img = um.make_image(h, w, c, seed=i)
        lens = _lens(lm.RADTAN, list(rad) + [0.0, 0.0, 0.0], tan)
        assert um.sha(gpu_ctx.undistort([img], K, lens=lens)[0]) == str(g[f"{name}/model_remap_sha"]), name
        xy, fr = gpu_ctx.undistort_map(w, h, K, lens=lens)
        assert um.sha(xy, fr) == um.sha(*um.model_maps_for(w, h, K, rad, tan)), name


def test_one_batched_call_mixes_models_sizes_and_channels(gpu_ctx, gold):
    """one l3d_undistort_u8 call over every lens case and two pinhole images, interleaved, on device memory: each output is the one
    image's own result, and the call launches one kernel per lens kind present (radtan, rational, fisheye)"""
    import torch
    g = np.load(PINHOLE_GOLDEN)
    items = [_case(gold, n) for n in _cases()]
    for i, name in enumerate(("tiny", "colmap_opencv")):
        w, h, c, K, rad, tan = um.case_params(g, name)
        items.insert(2 * i + 1, (um.make_image(h, w, c, seed=40 + i), K, _lens(lm.RADTAN, list(rad) + [0, 0, 0], tan)))
    descs = (capi.UndistortDesc * len(items))()
    dsts, keep = [], []
    for i, (img, K, lens) in enumerate(items):
        h, w = img.shape[:2]
        c = 1 if img.ndim == 2 else 3
        s = torch.from_numpy(img.reshape(h, w * c)).cuda()
        d = torch.full((h, w * c + 16), 77, dtype=torch.uint8, device="cuda")
        keep.append(s); dsts.append(d)
        descs[i] = capi.make_undistort_desc(w, h, c, K, src=s.data_ptr(), src_pitch=w * c, dst=d.data_ptr(), dst_pitch=w * c + 16,
                                            **capi.lens_desc_args(lens))
    before = gpu_ctx.launch_count()
    gpu_ctx.undistort_device(descs)
    gpu_ctx.sync()
    assert gpu_ctx.launch_count() == before + 3
    for (img, K, lens), d in zip(items, dsts):
        h, w = img.shape[:2]
        c = 1 if img.ndim == 2 else 3
        o = d.cpu().numpy()
        assert (o[:, w * c:] == 77).all()
        assert np.array_equal(o[:, :w * c].reshape(img.shape), gpu_ctx.undistort([img], K, lens=lens)[0])


def test_cpp_lens_overload_equals_the_c_abi(gpu_ctx, gold):
    """Line3D::undistortImage(in, out, LensDistortion, K) (through l3dpp_undistort_image_lens and line3d.undistort_image) gives the bytes
    of l3d_undistort_u8; a fisheye lens with a radtan-only term is rejected"""
    L = gpu_ctx.L
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    for name in ("fisheye_odd", "rational_odd", "fisheye_k"):
        img, K, lens = _case(gold, name)
        h, w = img.shape[:2]
        c = 1 if img.ndim == 2 else 3
        out = np.zeros_like(img)
        l9 = np.array([lens["model"]] + list(lens["k"]) + list(lens["p"]), np.float64)
        assert L.l3dpp_undistort_image_lens(p(img), p(out), h, w, c, p(l9), p(np.ascontiguousarray(K, np.float64)), 0) == 0
        ref = gpu_ctx.undistort([img], K, lens=lens)[0]
        assert np.array_equal(out, ref) and np.array_equal(line3d.undistort_image(img, K, lens), ref)
    img, K, _ = _case(gold, "fisheye_k")
    for bad in (_lens(1, [0.1, 0, 0, 0, 0.2, 0], [0, 0]), _lens(1, [0.1, 0, 0, 0, 0, 0], [0.01, 0]), _lens(2, [0] * 6, [0, 0])):
        with pytest.raises(ValueError):
            line3d.undistort_image(img, K, bad)


def test_rejected_lens_arguments(gpu_ctx):
    """unknown model, non-finite rational / fisheye terms, a fisheye descriptor with radial, tangential or rational terms: L3D_ERR_INVALID
    from l3d_undistort_u8 and l3d_undistort_map; l3d_remap_u8 does not use the camera"""
    L = gpu_ctx.L
    src, dst = np.zeros(64 * 48, np.uint8), np.zeros(64 * 48, np.uint8)
    xy, fr = np.zeros(64 * 48 * 2, np.int16), np.zeros(64 * 48, np.uint16)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    K = np.array([[50.0, 0, 32], [0, 50, 24], [0, 0, 1]])
    mk = lambda **kw: capi.make_undistort_desc(64, 48, 1, K, src=src.ctypes.data, dst=dst.ctypes.data, **kw)
    bad = {"model=2": dict(model=2), "model=-1": dict(model=-1), "k4=inf": dict(rational=(np.inf, 0, 0)), "k6=nan": dict(rational=(0, 0, np.nan)),
           "fisheye k2=nan": dict(model=1, fisheye=(0, np.nan, 0, 0)), "fisheye k4=inf (radtan)": dict(fisheye=(0, 0, 0, np.inf)),
           "fisheye+k1": dict(model=1, radial=(0.1, 0, 0)), "fisheye+k3": dict(model=1, radial=(0, 0, 0.1)),
           "fisheye+p1": dict(model=1, tangential=(0.01, 0)), "fisheye+k5": dict(model=1, rational=(0, 0.2, 0))}
    for what, kw in bad.items():
        d = mk(**kw)
        assert L.l3d_undistort_u8(gpu_ctx.h, 1, C.byref(d), 0) == -1, what
        assert L.l3d_undistort_map(gpu_ctx.h, C.byref(d), p(xy), p(fr), 0) == -1, what
        assert L.l3d_remap_u8(gpu_ctx.h, C.byref(d), p(xy), p(fr), 0) == 0, what
    for kw in (dict(model=1, fisheye=(0.1, 0.01, 0, 0)), dict(rational=(0.1, 0, 0)), dict(model=1, fisheye=(0.1, 0, 0, 0), radial=(-0.0, 0, 0))):
        d = mk(**kw)
        assert L.l3d_undistort_u8(gpu_ctx.h, 1, C.byref(d), 0) == 0, kw


def test_lens_calls_leave_the_pipeline_results_alone(gold):
    """a context holding matches, a score sweep and an affinity matrix gives the same view matches and diffusion result after fisheye and
    rational undistortion calls, successful and rejected"""
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
    img, K, fe = _case(gold, "fisheye_odd")
    _, _, ra = _case(gold, "rational_odd")
    ctx.undistort([img, img[:, :, 0].copy()], K, lens=[fe, ra])
    ctx.undistort_map(img.shape[1], img.shape[0], K, lens=fe)
    for bad in (_lens(7, [0] * 6, [0, 0]), _lens(1, [0.1, 0, 0, 0, 0, 0], [0.01, 0]), _lens(0, [0, 0, 0, np.nan, 0, 0], [0, 0])):
        with pytest.raises(capi.L3DError, match=r"failed \(-1\)"):
            ctx.undistort([img], K, lens=bad)
        with pytest.raises(capi.L3DError, match=r"failed \(-1\)"):
            ctx.undistort_map(img.shape[1], img.shape[0], K, lens=bad)
    assert results() == before
    ctx.close()
