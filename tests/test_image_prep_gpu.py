"""Image preparation for line detection on the GPU (l3d_prepare_gray_u8, Line3D::addImage with an image) against the numpy
restatement (tests/image_prep_model.py) and what OpenCV computed (tests/golden/ref_image_prep_v1.npz)."""
import ctypes as C
import os
import threading
import time

import numpy as np
import pytest

from line3dpp_b200 import capi, line3d
from tests import image_prep_model as pm
from tests import nvm_util as nu
from tests.test_image_prep_cpu import GOLDEN, case_image

pytestmark = pytest.mark.gpu

MW = 1920                       # max_img_width of the Line3D runs: 3072 x 2304 -> 1920 x 1440
VSFM = "rgb_vsfm_1920"          # the golden case of that size


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLDEN)


def _cases():
    return [str(n) for n in np.load(GOLDEN)["cases"]]


def _padded(img, pad):
    """img as a view into wider rows (row stride = row bytes + pad)"""
    if not pad:
        return img
    wide = np.zeros((img.shape[0], img.shape[1] + pad) + img.shape[2:], np.uint8)
    wide[:, :img.shape[1]] = img
    return wide[:, :img.shape[1]]


@pytest.mark.parametrize("name", _cases())
def test_kernel_equals_opencv_and_the_model(gpu_ctx, gold, name):
    img, mw, pad = case_image(gold, name)
    out = gpu_ctx.prepare_gray([_padded(img, pad)], mw)[0]
    assert [out.shape[1], out.shape[0]] == gold[f"{name}/out_size"].tolist()
    assert pm.sha(out) == str(gold[f"{name}/cv_sha"])
    assert np.array_equal(out, pm.prepare(img, mw))


def test_one_batched_call_over_every_case(gpu_ctx, gold):
    """one launch over every case (sizes, channel counts, max_img_width and modes mixed) on device memory with row pitches above the
    row's bytes; every output is cv2's, bytes beyond the rows are untouched, and host mode gives the same bytes"""
    import torch
    names = _cases()
    cases = [case_image(gold, n) for n in names]
    descs = (capi.ImagePrepDesc * len(cases))()
    dsts = []
    keep = []
    for i, (img, mw, pad) in enumerate(cases):
        h, w = img.shape[:2]
        c = 1 if img.ndim == 2 else 3
        ow, oh, _ = capi.image_prep_size(w, h, mw)
        sp, dp = w * c + pad + 3 * i, ow + 64 + i
        s = torch.zeros((h, sp), dtype=torch.uint8, device="cuda")
        s[:, :w * c] = torch.from_numpy(img.reshape(h, w * c)).cuda()
        d = torch.full((oh, dp), 77, dtype=torch.uint8, device="cuda")
        keep.append(s)
        dsts.append(d)
        descs[i] = capi.make_image_prep_desc(w, h, c, mw, s.data_ptr(), sp, d.data_ptr(), dp)
    before = gpu_ctx.launch_count()
    gpu_ctx.prepare_gray_device(descs)
    gpu_ctx.sync()
    assert gpu_ctx.launch_count() == before + 1
    dev = []
    for i, name in enumerate(names):
        ow, oh = gold[f"{name}/out_size"].tolist()
        o = dsts[i].cpu().numpy()
        assert (o[:, ow:] == 77).all(), f"{name}: bytes beyond the row were written"
        out = np.ascontiguousarray(o[:, :ow])
        assert pm.sha(out) == str(gold[f"{name}/cv_sha"]), name
        dev.append(out)
    host = gpu_ctx.prepare_gray([_padded(img, pad) for img, _, pad in cases], [mw for _, mw, _ in cases])
    for a, b in zip(host, dev):
        assert np.array_equal(a, b)


def test_every_rgb_triple(gpu_ctx, gold):
    """all 2^24 RGB triples as one 4096 x 4096 image (no resize) give the model's grey values, and the committed cv2 sample"""
    v = np.arange(1 << 24, dtype=np.uint32)
    rgb = np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    out = gpu_ctx.prepare_gray([rgb], -1)[0]
    assert np.array_equal(out, pm.gray(rgb))
    idx = gold["gray_rgb"].astype(np.int64)
    assert np.array_equal(out.reshape(-1)[(idx[:, 0] << 16) | (idx[:, 1] << 8) | idx[:, 2]], gold["gray_val"])


def test_rejected_arguments(gpu_ctx):
    L = gpu_ctx.L
    src, dst = np.zeros(64 * 48 * 3, np.uint8), np.zeros(64 * 48 * 3, np.uint8)

    def desc(**kw):
        a = dict(width=64, height=48, channels=3, mw=-1)
        a.update(kw)
        return capi.make_image_prep_desc(a["width"], a["height"], a["channels"], a["mw"], src.ctypes.data, None, dst.ctypes.data, None)

    bad = {"channels=2": desc(channels=2), "channels=4": desc(channels=4)}
    d = desc(); d.width = 0; bad["width=0"] = d
    d = desc(); d.height = 40000; bad["height=40000"] = d
    d = desc(); d.out_width = 63; bad["out_width"] = d
    d = desc(mw=32); d.out_height = 48; bad["out size without the resize"] = d
    d = desc(); d.src_pitch = 191; bad["src_pitch"] = d
    d = desc(); d.dst_pitch = 63; bad["dst_pitch"] = d
    d = desc(); d.src = None; bad["null src"] = d
    d = desc(); d.dst = None; bad["null dst"] = d
    d = desc(); d.dst = d.src; bad["src == dst"] = d
    for what, d in bad.items():
        assert L.l3d_prepare_gray_u8(gpu_ctx.h, 1, C.byref(d), 0) == -1, what
        assert L.l3d_last_error(gpu_ctx.h).decode().startswith("l3d_prepare_gray_u8:"), what
    assert L.l3d_prepare_gray_u8(gpu_ctx.h, -1, C.byref(desc()), 0) == -1
    assert L.l3d_prepare_gray_u8(gpu_ctx.h, 1, None, 0) == -1
    assert L.l3d_prepare_gray_u8(gpu_ctx.h, 0, None, 0) == 0
    assert L.l3d_prepare_gray_u8(gpu_ctx.h, 1, C.byref(desc(mw=32)), 0) == 0


# ------------------------------------------------------------------------------------------------ addImage with an image
@pytest.fixture(scope="module")
def inp():
    return nu.load_inputs()


@pytest.fixture(scope="module")
def image(gold):
    """the 3072 x 2304 RGB golden image; every view gets it (the detector decides the segments)"""
    img, mw, _ = case_image(gold, VSFM)
    assert mw == MW
    return img


def detections(inp, i):
    """what the detector returns for view i, in the prepared image's coordinates: the view's nvm segments scaled down, a repeat of
    some of them (equal lengths), and segments too short to survive"""
    s = inp["segs"][i].astype(np.float32)
    f = np.float32(MW) / np.float32(3072)
    short = np.array([[10, 10, 12, 11], [500, 400, 500, 405], [7, 7, 7, 7]], np.float32)
    return np.concatenate([s * f, s[::5] * f, short]).astype(np.float32)


def expected(inp, i, max_segments=3000):
    return pm.postprocess(detections(inp, i), 3072, 2304, MW, 1440, max_segments)


def _add(L, inp, i, img, segs=()):
    L.add_image_pixels(i, img, inp["K"][i], inp["R"][i], inp["t"][i], inp["median_depth"][i], inp["wps"][i], segs)


def test_detector_sees_the_prepared_image_and_the_cache_is_written(inp, image, gold, tmp_path):
    L = line3d.Line3D(True, True, output_folder=str(tmp_path), load_segments=True, max_img_width=MW)
    seen = []
    L.set_segment_detector(lambda g: (seen.append(g), detections(inp, 0))[1])
    _add(L, inp, 0, image)
    assert len(seen) == 1 and seen[0].shape == (1440, 1920)
    assert pm.sha(seen[0]) == str(gold[f"{VSFM}/cv_sha"])
    want = expected(inp, 0)
    assert 0 < len(want) < len(detections(inp, 0))
    assert L.view_segments(0).tobytes() == want.tobytes()
    path = line3d.segment_cache_path(str(tmp_path), 0, 3072, 2304, MW)
    line3d.write_segment_cache(tmp_path / "same.bin", want)
    assert open(path, "rb").read() == (tmp_path / "same.bin").read_bytes()
    L.close()
    # a second Line3D on the same folder reads the cache and never calls its detector
    L2 = line3d.Line3D(True, True, output_folder=str(tmp_path), load_segments=True, max_img_width=MW)

    def must_not_run(_):
        raise AssertionError("the detector ran although the segment cache exists")
    L2.set_segment_detector(must_not_run)
    _add(L2, inp, 0, image)
    assert L2.view_segments(0).tobytes() == want.tobytes()
    L2.close()


def test_cut_at_max_line_segments(inp, image, tmp_path):
    for devices in (None, [0]):                  # the device-list constructor takes max_line_segments as well
        L = line3d.Line3D(True, True, output_folder=str(tmp_path), load_segments=False, max_img_width=MW, max_line_segments=500, devices=devices)
        L.set_segment_detector(lambda g: detections(inp, 1))
        _add(L, inp, 1, image)
        assert L.view_segments(1).tobytes() == expected(inp, 1, 500).tobytes(), devices
        L.close()


def test_without_load_segments_nothing_is_written(inp, image, tmp_path):
    L = line3d.Line3D(True, True, output_folder=str(tmp_path), load_segments=False, max_img_width=MW)
    calls = []
    L.set_segment_detector(lambda g: (calls.append(1), detections(inp, 2))[1])
    _add(L, inp, 2, image)
    assert calls == [1] and os.listdir(tmp_path) == []
    assert L.view_segments(2).tobytes() == expected(inp, 2).tobytes()
    L.close()


def test_rejected_views(inp, image, tmp_path):
    L = line3d.Line3D(True, True, output_folder=str(tmp_path), load_segments=True, max_img_width=MW)
    with pytest.raises(capi.L3DError, match="no line segments given and no segment cache .*segments_L3D\\+\\+_0_1920x1440_3000.bin"):
        _add(L, inp, 0, image)                                           # no detector: the message of the size overload
    L.set_segment_detector(lambda g: False)
    with pytest.raises(capi.L3DError, match="segment detector failed"):
        _add(L, inp, 0, image)
    L.set_segment_detector(lambda g: np.array([[1, 1, 3, 3], [9, 9, 9, 15]], np.float32))
    with pytest.raises(capi.L3DError, match="none of the 2 detected segments is longer"):
        _add(L, inp, 0, image)
    with pytest.raises(KeyError):
        L.view_segments(0)
    assert not os.path.exists(tmp_path / "L3D++_data")
    # 4 channels: only through the C wrapper (the Python side accepts HxW and HxWx3)
    px = np.zeros((900, 1000, 4), np.uint8)
    f64 = lambda a: np.ascontiguousarray(a, np.float64).ctypes.data_as(C.c_void_p)
    wps = np.ascontiguousarray(inp["wps"][0], np.uint32)
    rc = L.L.l3dpp_add_image_pixels(L.h, 0, px.ctypes.data_as(C.c_void_p), 900, 1000, 4, C.c_longlong(4000), f64(inp["K"][0]), f64(inp["R"][0]),
                                    f64(inp["t"][0]), C.c_float(1.0), wps.ctypes.data_as(C.c_void_p), len(wps), None, 0)
    assert rc == -1 and "image type not supported: 4 channels" in L.L.l3dpp_last_error(L.h).decode()
    L.close()


def test_views_that_never_reach_the_detector(inp, image, tmp_path):
    L = line3d.Line3D(True, True, output_folder=str(tmp_path), load_segments=True, max_img_width=MW)
    calls = []
    L.set_segment_detector(lambda g: (calls.append(g.shape), detections(inp, 3))[1])
    segs = inp["segs"][3]
    _add(L, inp, 3, image, segs)                                         # explicit segments are used as given
    assert L.view_segments(3).tobytes() == np.ascontiguousarray(segs, np.float32).tobytes()
    with pytest.raises(capi.L3DError, match="camera ID already in use"):
        _add(L, inp, 3, image)
    with pytest.raises(capi.L3DError, match="too small"):
        _add(L, inp, 4, image[:799, :799])
    assert calls == [] and not os.path.exists(tmp_path / "L3D++_data")
    L.close()


def test_concurrent_calls_equal_a_serial_run(inp, image, tmp_path):
    """eight Python threads calling add_image_pixels at once (ctypes drops the GIL, the detector sleeps outside it) give the views
    of a serial run; the detectors really overlap"""
    views = list(range(16))
    state = threading.local()
    active, peak, lock = [0], [0], threading.Lock()

    def detector(g):
        with lock:
            active[0] += 1
            peak[0] = max(peak[0], active[0])
        time.sleep(0.05)
        with lock:
            active[0] -= 1
        state.seen = pm.sha(g)
        return detections(inp, state.view)

    def run(folder, threads):
        os.makedirs(folder)
        L = line3d.Line3D(True, True, output_folder=str(folder), load_segments=True, max_img_width=MW)
        L.set_segment_detector(detector)
        seen = {}

        def work(vs):
            for v in vs:
                state.view = v
                _add(L, inp, v, image)
                seen[v] = state.seen
        parts = [views[k::threads] for k in range(threads)]
        ts = [threading.Thread(target=work, args=(p,)) for p in parts]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        out = {v: L.view_segments(v).tobytes() for v in views}
        L.close()
        return out, seen

    serial, seen_serial = run(tmp_path / "serial", 1)
    peak[0] = 0
    par, seen_par = run(tmp_path / "threads", 8)
    assert peak[0] > 1
    assert par == serial and seen_par == seen_serial
    assert all(serial[v] == expected(inp, v).tobytes() for v in views)
    files = sorted(os.listdir(tmp_path / "serial" / "L3D++_data"))
    assert len(files) == len(views) and sorted(os.listdir(tmp_path / "threads" / "L3D++_data")) == files
    for f in files:
        assert (tmp_path / "threads" / "L3D++_data" / f).read_bytes() == (tmp_path / "serial" / "L3D++_data" / f).read_bytes()


def test_full_pipeline_through_the_image_path(inp, image, tmp_path):
    """a reconstruction fed through addImage with images and the detector equals the one fed the resulting segments directly:
    the same match lists, 3D segments and residuals, bit for bit"""
    def run(with_images):
        L = line3d.Line3D(True, True, output_folder=str(tmp_path), load_segments=False, max_img_width=MW)
        L.set_segment_detector(lambda g: detections(inp, run.view))
        for i in range(inp["V"]):
            if with_images:
                run.view = i
                _add(L, inp, i, image)
            else:
                w, h = inp["wh"][i]
                L.add_image(i, int(w), int(h), inp["K"][i], inp["R"][i], inp["t"][i], inp["median_depth"][i], inp["wps"][i], expected(inp, i))
        L.match_images()
        L.reconstruct_3d_lines(3, False)
        matches = [L.view_matches(i, False).tobytes() for i in range(inp["V"])]
        digest = pm.sha(L.segments3d(), L.residuals())             # every field, doubles bit for bit
        st = L.stats()
        L.close()
        return matches, digest, st

    a, b = run(True), run(False)
    assert a[2]["lines3D"] > 100
    assert a[0] == b[0] and a[1] == b[1]
    assert {k: v for k, v in a[2].items() if not k.startswith("ms_")} == {k: v for k, v in b[2].items() if not k.startswith("ms_")}
