"""Undistortion into a new camera matrix and size on the GPU (l3d_undistort_desc's new_fx .. out_height; DESIGN.md §4a): the maps
against cv2's (tests/golden/ref_undistort_newk_v1.npz) and the restatement (tests/newk_model.py), the fused kernel against the remap of
its own map, a zero tail and newK = K against today's bytes, mixed batches, every new rejection, and the C++, C-wrapper and Python
entry points."""
import ctypes as C
import os

import numpy as np
import pytest

from line3dpp_b200 import capi, line3d
from tests import lens_model as lm
from tests import newk_model as nm
from tests import undistort_model as um

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "ref_undistort_newk_v1.npz")
LENS_GOLDEN = os.path.join(HERE, "golden", "ref_undistort_lens_v1.npz")
PINHOLE_GOLDEN = os.path.join(HERE, "golden", "ref_undistort_v1.npz")
# as for the lens models (tests/test_undistort_lens_gpu.py): the device's atan may differ from glibc's in the last ulp, which can move
# a fisheye u or v across a rounding boundary; at most this many entries per million beyond the restatement's own count
FISHEYE_EXTRA_PER_MILLION = 20


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLDEN)


def _cases(model=None):
    g = np.load(GOLDEN)
    return [str(n) for n in g["cases"] if model is None or int(g[f"{n}/model"]) == model]


def _case(g, name):
    """(image, K, lens, newK, out_size) of a golden case"""
    w, h, c, K, model, k, p, newK, out_size = nm.case_params(g, name)
    return um.make_image(h, w, c, seed=200 + _cases().index(name)), K, nm.lens_dict(model, k, p), newK, out_size


def _fixed(xy, fr):
    return xy[..., 0].astype(np.int64) * 32 + (fr & 31), xy[..., 1].astype(np.int64) * 32 + (fr >> 5)


@pytest.mark.parametrize("name", _cases())
def test_map_is_within_one_step_of_opencv(gpu_ctx, gold, name):
    img, K, lens, newK, (ow, oh) = _case(gold, name)
    h, w = img.shape[:2]
    xy, fr = gpu_ctx.undistort_map(w, h, K, lens=lens, new_K=newK, out_size=(ow, oh))
    assert xy.shape == (oh, ow, 2)
    mxy, mfr = nm.newk_maps(ow, oh, K, newK, lens["model"], lens["k"], lens["p"])
    if lens["model"] == lm.RADTAN:              # plain IEEE operations: the restatement's map exactly
        assert np.array_equal(xy, mxy) and np.array_equal(fr, mfr)
    cxy, cfr = um.apply_corrections(mxy, mfr, gold[f"{name}/diff_idx"], gold[f"{name}/diff_xy"], gold[f"{name}/diff_frac"])
    assert um.sha(cxy, cfr) == str(gold[f"{name}/cv_map_sha"])
    (gu, gv), (cu, cv) = _fixed(xy, fr), _fixed(cxy, cfr)
    du, dv = np.abs(gu - cu), np.abs(gv - cv)
    du, dv = np.minimum(du, 65536 * 32 - du), np.minimum(dv, 65536 * 32 - dv)   # fisheye_int16: compare modulo the wrap
    assert du.max() <= 1 and dv.max() <= 1
    differ = int(((du != 0) | (dv != 0)).sum())
    model_differ = len(gold[f"{name}/diff_idx"])
    print(f"{name}: {differ} of {ow * oh} map entries differ from cv2's (restatement: {model_differ})")
    assert differ <= model_differ + FISHEYE_EXTRA_PER_MILLION * ow * oh // 1_000_000 + (lens["model"] == lm.FISHEYE)


@pytest.mark.parametrize("name", _cases())
def test_fused_output_is_the_remap_of_its_own_map(gpu_ctx, gold, name):
    img, K, lens, newK, out_size = _case(gold, name)
    h, w = img.shape[:2]
    xy, fr = gpu_ctx.undistort_map(w, h, K, lens=lens, new_K=newK, out_size=out_size)
    fused = gpu_ctx.undistort([img], K, lens=lens, new_K=newK, out_size=out_size)[0]
    assert fused.shape == (out_size[1], out_size[0]) + img.shape[2:]
    assert np.array_equal(fused, gpu_ctx.remap(img, xy, fr))
    if lens["model"] == lm.RADTAN:
        assert um.sha(fused) == str(gold[f"{name}/model_remap_sha"])
        if not len(gold[f"{name}/diff_idx"]):
            assert um.sha(fused) == str(gold[f"{name}/cv_remap_sha"])


def test_zero_tail_and_new_k_equal_to_k_give_todays_bytes(gpu_ctx):
    """every case of the pinhole and lens goldens: the zero tail, and newK = K with out size = source, give the stored bytes"""
    g, gl = np.load(PINHOLE_GOLDEN), np.load(LENS_GOLDEN)
    items = []
    for i, name in enumerate(str(n) for n in g["cases"]):
        w, h, c, K, rad, tan = um.case_params(g, name)
        items.append((um.make_image(h, w, c, seed=i), K, nm.lens_dict(0, list(rad) + [0, 0, 0], tan), str(g[f"{name}/model_remap_sha"])))
    lens_names = [str(n) for n in gl["cases"]]
    for i, name in enumerate(lens_names):
        w, h, c, K, model, k, p = lm.case_params(gl, name)
        if model == lm.RADTAN:
            items.append((um.make_image(h, w, c, seed=100 + i), K, nm.lens_dict(model, k, p), str(gl[f"{name}/model_remap_sha"])))
    for img, K, lens, sha in items:
        h, w = img.shape[:2]
        a = gpu_ctx.undistort([img], K, lens=lens)[0]
        b = gpu_ctx.undistort([img], K, lens=lens, new_K=K, out_size=(w, h))[0]
        assert um.sha(a) == sha and um.sha(b) == sha
    for i, name in enumerate(lens_names):          # fisheye: the zero tail and newK = K agree, maps and images
        w, h, c, K, model, k, p = lm.case_params(gl, name)
        if model != lm.FISHEYE:
            continue
        lens, img = nm.lens_dict(model, k, p), um.make_image(h, w, c, seed=100 + i)
        m0 = gpu_ctx.undistort_map(w, h, K, lens=lens)
        m1 = gpu_ctx.undistort_map(w, h, K, lens=lens, new_K=K, out_size=(w, h))
        assert um.sha(*m0) == um.sha(*m1)
        assert np.array_equal(gpu_ctx.undistort([img], K, lens=lens)[0], gpu_ctx.undistort([img], K, lens=lens, new_K=K, out_size=(w, h))[0])


@pytest.mark.parametrize("on_device", [True, False])
def test_one_batch_mixes_kinds_sizes_channels_and_new_ks(gpu_ctx, gold, on_device):
    """one l3d_undistort_u8 call over every golden case interleaved with the same images without a new K: each output is the image's
    own single-call result; the device-mode outputs keep their row padding"""
    import torch
    items = []
    for name in _cases():
        img, K, lens, newK, out_size = _case(gold, name)
        if img.size > 2_000_000:
            img, K = img[:700, :900].copy(), K           # a crop: the batch stays small; the maps do not depend on the source size
        items += [(img, K, lens, newK, out_size), (img, K, lens, None, None)]
    n = len(items)
    refs = [gpu_ctx.undistort([img], K, lens=lens, new_K=nk, out_size=os_)[0] for img, K, lens, nk, os_ in items]
    if not on_device:
        outs = gpu_ctx.undistort([it[0] for it in items], [it[1] for it in items], lens=[it[2] for it in items], new_K=[it[3] for it in items],
                                 out_size=[it[4] for it in items])
        for o, r in zip(outs, refs):
            assert np.array_equal(o, r)
        return
    descs = (capi.UndistortDesc * n)()
    dsts, keep = [], []
    for i, (img, K, lens, nk, os_) in enumerate(items):
        h, w = img.shape[:2]
        c = 1 if img.ndim == 2 else 3
        ow, oh = (w, h) if os_ is None else os_
        s = torch.from_numpy(img.reshape(h, w * c)).cuda()
        d = torch.full((oh, ow * c + 16), 77, dtype=torch.uint8, device="cuda")
        keep.append(s); dsts.append(d)
        descs[i] = capi.make_undistort_desc(w, h, c, K, src=s.data_ptr(), src_pitch=w * c, dst=d.data_ptr(), dst_pitch=ow * c + 16, new_K=nk,
                                            out_size=os_, **capi.lens_desc_args(lens))
    gpu_ctx.undistort_device(descs)
    gpu_ctx.sync()
    for (img, K, lens, nk, os_), d, r in zip(items, dsts, refs):
        c = 1 if img.ndim == 2 else 3
        o = d.cpu().numpy()
        assert (o[:, r.shape[1] * c:] == 77).all()
        assert np.array_equal(o[:, :r.shape[1] * c].reshape(r.shape), r)


def test_rejected_new_k_and_size(gpu_ctx):
    """a new K with fx' or fy' zero or not finite, or cx' or cy' not finite; an output size other than (0, 0) outside [1, 32767]; a dst
    pitch below out_width * channels: L3D_ERR_INVALID from the calls that use them"""
    L = gpu_ctx.L
    src, dst = np.zeros(64 * 48, np.uint8), np.zeros(100 * 80, np.uint8)
    xy, fr = np.zeros(100 * 80 * 2, np.int16), np.zeros(100 * 80, np.uint16)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    K = np.array([[50.0, 0, 32], [0, 50, 24], [0, 0, 1]])
    mk = lambda **kw: capi.make_undistort_desc(64, 48, 1, K, src=src.ctypes.data, dst=dst.ctypes.data, **kw)
    nK = lambda fx, fy, cx, cy: np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]])
    bad_k = {"fx'=0": nK(0, 40, 30, 20), "fy'=0": nK(40, 0, 30, 20), "fx'=inf": nK(np.inf, 40, 30, 20), "fy'=nan": nK(40, np.nan, 30, 20),
             "cx'=nan": nK(40, 40, np.nan, 20), "cy'=-inf": nK(40, 40, 30, -np.inf), "K'=(0, 0, 1, 0)": nK(0, 0, 1, 0)}
    bad_size = {"(0, 10)": (0, 10), "(10, 0)": (10, 0), "(-1, -1)": (-1, -1), "(32768, 10)": (32768, 10), "(10, 32768)": (10, 32768)}
    for what, kw in [(k, dict(new_K=v)) for k, v in bad_k.items()] + [(k, dict(out_size=v)) for k, v in bad_size.items()]:
        d = mk(**kw)
        assert L.l3d_undistort_u8(gpu_ctx.h, 1, C.byref(d), 0) == -1, what
        assert L.l3d_undistort_map(gpu_ctx.h, C.byref(d), p(xy), p(fr), 0) == -1, what
        if "out_size" in kw:
            assert L.l3d_remap_u8(gpu_ctx.h, C.byref(d), p(xy), p(fr), 0) == -1, what
        else:                                   # the remap does not use the camera
            assert L.l3d_remap_u8(gpu_ctx.h, C.byref(d), p(xy), p(fr), 0) == 0, what
    d = mk(out_size=(100, 80), dst_pitch=99)
    for rc in (L.l3d_undistort_u8(gpu_ctx.h, 1, C.byref(d), 0), L.l3d_remap_u8(gpu_ctx.h, C.byref(d), p(xy), p(fr), 0)):
        assert rc == -1
    for ok in (dict(new_K=nK(40, 41, 0, 0)), dict(new_K=nK(-40, 40, 30, 20)), dict(out_size=(1, 1)), dict(out_size=(100, 80), new_K=nK(60, 60, 50, 40))):
        d = mk(**ok)
        assert L.l3d_undistort_u8(gpu_ctx.h, 1, C.byref(d), 0) == 0, ok
    img, K2 = um.make_image(48, 64, 1, seed=3), K
    with pytest.raises(ValueError):
        line3d.undistort_image(img, K2, nm.lens_dict(0, [0.1, 0, 0, 0, 0, 0], [0, 0]), new_K=nK(0, 40, 30, 20))
    with pytest.raises(ValueError):
        line3d.undistort_image(img, K2, nm.lens_dict(0, [0.1, 0, 0, 0, 0, 0], [0, 0]), out_size=(0, 10))


def test_cpp_c_wrapper_and_python_entry_points(gpu_ctx, gold):
    """Line3D::undistortImage(in, out, lens, K, newK, w, h) through l3dpp_undistort_image_newk and line3d.undistort_image gives the
    bytes of l3d_undistort_u8, with newK from the host functions; the older overloads are the zero tail"""
    L = gpu_ctx.L
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    for name in ("radtan5_a05_smaller", "rational8_a1_nonprop", "fisheye_b05_smaller", "fisheye_b1_larger_nonprop"):
        img, K, lens, newK, (ow, oh) = _case(gold, name)
        h, w = img.shape[:2]
        c = 1 if img.ndim == 2 else 3
        ref = gpu_ctx.undistort([img], K, lens=lens, new_K=newK, out_size=(ow, oh))[0]
        out = np.zeros((oh, ow) + img.shape[2:], np.uint8)
        l9 = np.array([lens["model"]] + list(lens["k"]) + list(lens["p"]), np.float64)
        assert L.l3dpp_undistort_image_newk(p(img), p(out), h, w, c, p(l9), p(np.ascontiguousarray(K, np.float64)),
                                            p(np.ascontiguousarray(newK, np.float64)), oh, ow, 0) == 0
        assert np.array_equal(out, ref)
        assert np.array_equal(line3d.undistort_image(img, K, lens, new_K=newK, out_size=(ow, oh)), ref)
        assert np.array_equal(line3d.undistort_image(img, K, lens), gpu_ctx.undistort([img], K, lens=lens)[0])
    img, K, lens, _, _ = _case(gold, "radtan5_a0")
    newK, roi = line3d.optimal_new_camera_matrix(K, lens, (img.shape[1], img.shape[0]), 1.0, (900, 700))
    assert np.array_equal(line3d.undistort_image(img, K, lens, new_K=newK, out_size=(900, 700)),
                          gpu_ctx.undistort([img], K, lens=lens, new_K=newK, out_size=(900, 700))[0])
