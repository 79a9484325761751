"""l3d_undistort_points on the GPU against what OpenCV 4.13 computed (tests/golden/ref_undistort_points_v1.npz), its rejections, and the
addImage overloads that take a lens: byte for byte what undistortImage / undistortPoints followed by the plain addImage give."""
import os

import numpy as np
import pytest

from line3dpp_b200 import capi, line3d, synth
from tests import nvm_util as nu
from tests import undistort_model as um
from tests import undistort_points_model as m

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "ref_undistort_points_v1.npz")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLDEN)


def _cases(model):
    g = np.load(GOLDEN)
    return [str(n) for n in g["cases"] if int(g[f"{n}/model"]) == model]


def _set(g, name):
    """(points, K, lens dict, new K or None, cv2's output) of a golden case"""
    P = f"{name}/"
    nK = g[P + "new_K"]
    lens = dict(model=int(g[P + "model"]), k=g[P + "k"], p=g[P + "p"])
    return g[P + "pts"], g[P + "K"], lens, (nK if np.any(nK) else None), g[P + "cv"]


def _ulps(a, b):
    """float32 ulp distance per entry (NaN against NaN: 0)"""
    ia = a.view(np.int32).astype(np.int64)
    ib = b.view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    d = np.abs(ia - ib)
    return np.where(np.isnan(a) & np.isnan(b), 0, d)


@pytest.mark.parametrize("name", _cases(m.RADTAN))
def test_radtan_is_bit_identical_to_opencv(gpu_ctx, gold, name):
    pts, K, lens, nK, cv = _set(gold, name)
    out, = gpu_ctx.undistort_points([(pts, K, lens, nK)])
    assert m.same(out, cv), np.flatnonzero(_ulps(out, cv).max(axis=1))[:10]


@pytest.mark.parametrize("name", _cases(m.RADTAN)[:2] + _cases(m.FISHEYE)[:1])
def test_device_mode_equals_host_mode(gpu_ctx, gold, name):
    import torch
    pts, K, lens, nK, cv = _set(gold, name)
    host, = gpu_ctx.undistort_points([(pts, K, lens, nK)])
    src = torch.from_numpy(np.ascontiguousarray(pts)).cuda()
    dst = torch.empty_like(src)
    torch.cuda.synchronize()
    gpu_ctx.undistort_points([(src, K, lens, nK)], out=[dst])
    gpu_ctx.sync()
    assert m.same(dst.cpu().numpy(), host)
    if lens["model"] == m.RADTAN:
        assert m.same(host, cv)


@pytest.mark.parametrize("name", _cases(m.FISHEYE))
def test_fisheye_equals_opencv_up_to_the_device_tan(gpu_ctx, gold, name):
    """where the device's tan and glibc's differ, the float32 output may be one ulp off; everything else, the failure value and NaN
    included, is OpenCV's"""
    pts, K, lens, nK, cv = _set(gold, name)
    out, = gpu_ctx.undistort_points([(pts, K, lens, nK)])
    d = _ulps(out, cv)
    assert d.max() <= 1, (name, int(d.max()))
    assert np.array_equal(np.isnan(out), np.isnan(cv)) and np.array_equal(out == m.FAIL, cv == m.FAIL)
    print(f"{name}: {int((d > 0).any(axis=1).sum())} of {len(pts)} points one ulp from OpenCV (device tan)")


def test_one_mixed_batch_of_every_case(gpu_ctx, gold):
    """every case in one launch, in an interleaved order with empty sets between them, gives what each set gives alone"""
    names = [str(n) for n in gold["cases"]]
    order = names[::2] + names[1::2]
    sets, alone = [], []
    for n in order:
        pts, K, lens, nK, cv = _set(gold, n)
        sets += [(pts, K, lens, nK), (np.zeros((0, 2), np.float32), K, lens, None)]
        alone.append(gpu_ctx.undistort_points([(pts, K, lens, nK)])[0])
    outs = gpu_ctx.undistort_points(sets)
    for i, n in enumerate(order):
        assert m.same(outs[2 * i], alone[i]), n
        if int(gold[f"{n}/model"]) == m.RADTAN:
            assert m.same(outs[2 * i], gold[f"{n}/cv"]), n
        assert outs[2 * i + 1].shape == (0, 2)
    # the same batch through Line3D::undistortPoints (a context of its own on the calling thread's device)
    again = line3d.undistort_points_batch([s for s in sets])
    for i in range(len(order)):
        assert m.same(again[2 * i], alone[i])


def test_in_place(gpu_ctx, gold):
    import torch
    pts, K, lens, nK, cv = _set(gold, "radtan8_opt")
    a = np.ascontiguousarray(pts).copy()
    gpu_ctx.undistort_points([(a, K, lens, nK)], out=[a])
    assert m.same(a, cv)
    t = torch.from_numpy(np.ascontiguousarray(pts)).cuda()
    torch.cuda.synchronize()
    gpu_ctx.undistort_points([(t, K, lens, nK)], out=[t])
    gpu_ctx.sync()
    assert m.same(t.cpu().numpy(), cv)
    segs = pts[: len(pts) // 2 * 2].reshape(-1, 4)
    assert m.same(line3d.undistort_points(segs, K, lens, nK).reshape(-1, 2), cv[: len(segs) * 2])


def test_rejections_name_the_reason_and_write_nothing(gpu_ctx):
    K = np.array([[900.0, 0, 640], [0, 910, 480], [0, 0, 1]])
    pts = np.arange(20, dtype=np.float32).reshape(10, 2)
    out = np.full_like(pts, 7.0)
    radtan = dict(model=m.RADTAN, k=(0.1, 0, 0, 0, 0, 0), p=(0, 0))
    fish = dict(model=m.FISHEYE, k=(0.1, 0, 0, 0), p=(0, 0))

    def desc(Km=K, lens=radtan, count=10, src=pts.ctypes.data, dst=out.ctypes.data, new_K=None):
        return capi.make_points_desc(Km, lens, count, src, dst, new_K)

    bad_K = np.array(K)
    bad_K[0, 0] = 0
    nan_K = np.array(K)
    nan_K[1, 2] = np.nan
    cases = [
        (desc(Km=bad_K), "fx and fy must be finite and non-zero"),
        (desc(Km=nan_K), "principal point and coefficients must be finite"),
        (desc(lens=dict(model=5)), "unknown lens model"),
        (desc(lens=dict(model=m.FISHEYE, k=(0.1, 0, 0, 0, 0.2, 0))), "a fisheye lens takes no radial, tangential or rational coefficients"),
        (desc(new_K=np.diag([0.0, 900.0, 1.0])), "new_fx and new_fy must be finite and non-zero"),
        (desc(new_K=np.array([[900.0, 0, np.inf], [0, 900, 0], [0, 0, 1]])), "new_cx and new_cy must be finite"),
        (desc(count=-1), "set 1: count < 0"),
        (desc(src=0), "set 1: null point pointer"),
        (desc(dst=0), "set 1: null point pointer"),
    ]
    for d, why in cases:
        arr = (capi.PointsDesc * 2)(desc(lens=fish), d)
        for on_device in (0, 1):
            with pytest.raises(capi.L3DError, match="l3d_undistort_points: " + why.replace("(", r"\(").replace(")", r"\)")):
                gpu_ctx.undistort_points_descs(arr, on_device)
            assert (out == 7.0).all(), why
    L = capi.lib()
    assert L.l3d_undistort_points(gpu_ctx.h, -1, None, 0) == -1
    assert L.l3d_undistort_points(gpu_ctx.h, 1, None, 0) == -1
    assert L.l3d_undistort_points(gpu_ctx.h, 0, None, 0) == 0
    # a rejected lens through the C++ helper is std::invalid_argument (ValueError here), naming the reason
    with pytest.raises(ValueError, match="undistortPoints: l3d_undistort_points: fx and fy must be finite and non-zero"):
        line3d.undistort_points(pts, bad_K, radtan)
    with pytest.raises(ValueError, match="pairs"):
        line3d.undistort_points_batch([(np.zeros(3, np.float32), K, radtan, None)])


# ------------------------------------------------------------------------------------------------ addImage with a lens
W, H = 1600, 1200
K0 = np.array([[1150.0, 0, 801.5], [0, 1160.0, 597.25], [0, 0, 1]])
LENSES = {"radtan": dict(model=m.RADTAN, k=(-0.18, 0.06, 0.0, 0, 0, 0), p=(0.0009, -0.0006)),
          "rational": dict(model=m.RADTAN, k=(0.12, -0.05, 0.01, 0.08, -0.02, 0.005), p=(0.0007, -0.0004)),
          "fisheye": dict(model=m.FISHEYE, k=(0.05, -0.01, 0.003, -0.0005), p=(0, 0))}
R0, T0 = np.eye(3), np.array([0.1, -0.2, 1.5])


def _detector(seen):
    """records the grey image it is given; detections derived from it, so that different inputs would give different segments"""
    def det(gray):
        seen.append(gray)
        h, w = gray.shape
        rows = np.arange(0, h - 8, 7)
        v = gray[rows, :].astype(np.float32).mean(axis=1)
        return np.stack([np.full_like(v, 3.0), rows.astype(np.float32), w - 3.0 - v, rows + v / 64], 1).astype(np.float32)
    return det


def _line3d(folder, mw):
    return line3d.Line3D(True, True, output_folder=str(folder), load_segments=True, max_img_width=mw)


@pytest.mark.parametrize("lens_name", list(LENSES))
@pytest.mark.parametrize("channels", [1, 3])
@pytest.mark.parametrize("mw", [-1, 1000])
def test_add_image_with_a_lens_equals_undistort_image_then_add_image(tmp_path, lens_name, channels, mw):
    lens = LENSES[lens_name]
    img = um.make_image(H, W, channels, seed=3 + channels)
    # the two-step loop: undistortImage, then addImage
    seen_a, seen_b = [], []
    os.makedirs(tmp_path / "a")
    os.makedirs(tmp_path / "b")
    A = _line3d(tmp_path / "a", mw)
    A.set_segment_detector(_detector(seen_a))
    A.add_image_pixels(5, line3d.undistort_image(img, K0, lens), K0, R0, T0, 2.0, [1, 2, 3])
    B = _line3d(tmp_path / "b", mw)
    B.set_segment_detector(_detector(seen_b))
    B.add_image_pixels(5, img, K0, R0, T0, 2.0, [1, 2, 3], lens=lens)
    assert len(seen_a) == len(seen_b) == 1
    assert seen_a[0].shape == seen_b[0].shape and seen_a[0].tobytes() == seen_b[0].tobytes()
    assert len(A.view_segments(5)) > 10
    assert A.view_segments(5).tobytes() == B.view_segments(5).tobytes()
    pa = line3d.segment_cache_path(str(tmp_path / "a"), 5, W, H, mw)
    pb = line3d.segment_cache_path(str(tmp_path / "b"), 5, W, H, mw)
    assert open(pa, "rb").read() == open(pb, "rb").read()
    # a cache hit: the stored segments as they are, no detector and no GPU work
    C2 = _line3d(tmp_path / "b", mw)

    def must_not_run(_):
        raise AssertionError("the detector ran although the segment cache exists")
    C2.set_segment_detector(must_not_run)
    C2.add_image_pixels(5, img, K0, R0, T0, 2.0, [1, 2, 3], lens=lens)
    assert C2.view_segments(5).tobytes() == B.view_segments(5).tobytes()
    for L in (A, B, C2):
        L.close()


def test_given_segments_and_the_zero_lens(tmp_path):
    inp = nu.load_inputs()
    segs = inp["segs"][0].astype(np.float32)
    K = inp["K"][0]
    img = um.make_image(2304, 3072, 1, seed=9)
    for lens in LENSES.values():
        want = line3d.undistort_points(segs, K, lens)
        for form in ("size", "image"):
            A = line3d.Line3D(True, True)
            B = line3d.Line3D(True, True)
            A.add_image(0, 3072, 2304, K, inp["R"][0], inp["t"][0], 2.0, inp["wps"][0], want)
            if form == "size":
                B.add_image(0, 3072, 2304, K, inp["R"][0], inp["t"][0], 2.0, inp["wps"][0], segs, lens=lens)
            else:
                B.add_image_pixels(0, img, K, inp["R"][0], inp["t"][0], 2.0, inp["wps"][0], segs, lens=lens)
            assert A.view_segments(0).tobytes() == B.view_segments(0).tobytes()
            A.close()
            B.close()
    # an all-zero lens is the plain overload: no undistortion (and no lens check)
    zero = dict(model=m.RADTAN, k=(0,) * 6, p=(0, 0))
    A = line3d.Line3D(True, True)
    A.add_image(0, 3072, 2304, K, inp["R"][0], inp["t"][0], 2.0, inp["wps"][0], segs, lens=zero)
    assert A.view_segments(0).tobytes() == segs.tobytes()
    A.close()


def test_rejected_lens_sets_last_error(tmp_path):
    inp = nu.load_inputs()
    segs = inp["segs"][0].astype(np.float32)
    L = line3d.Line3D(True, True, output_folder=str(tmp_path))
    bad = dict(model=m.FISHEYE, k=(0.1, 0, 0, 0, 0.5, 0), p=(0, 0))
    with pytest.raises(capi.L3DError, match=r"addImage \[0\]: lens: l3d_undistort_points: a fisheye lens takes no radial"):
        L.add_image(0, 3072, 2304, inp["K"][0], inp["R"][0], inp["t"][0], 2.0, inp["wps"][0], segs, lens=bad)
    bad_K = np.array(inp["K"][0])
    bad_K[1, 1] = np.inf
    L.set_segment_detector(lambda g: (_ for _ in ()).throw(AssertionError("the detector must not run")))
    with pytest.raises(capi.L3DError, match=r"addImage \[1\]: lens: l3d_undistort_points: fx and fy must be finite and non-zero"):
        L.add_image_pixels(1, um.make_image(900, 1000, 1), bad_K, inp["R"][0], inp["t"][0], 2.0, inp["wps"][0], lens=LENSES["radtan"])
    assert L.L.l3dpp_view_segments(L.h, 0, None, 0) == -1 and L.L.l3dpp_view_segments(L.h, 1, None, 0) == -1
    L.close()


def test_scene_with_distorted_segments_reconstructs_as_the_two_step_calls(tmp_path):
    """a synthetic scene whose segments are taken as detected in distorted images: addImage(..., lens) and addImage of the segments
    undistortPoints gives reconstruct the same 3D lines bit for bit"""
    sc = synth.make_scene(8, 200, 5, "ring2")
    lens = dict(model=m.RADTAN, k=(-0.02, 0.004, 0, 0, 0, 0), p=(0.0002, -0.0001))
    A = line3d.Line3D(neighbors_by_worldpoints=False)
    B = line3d.Line3D(neighbors_by_worldpoints=False)
    for i in range(sc.num_views):
        args = (sc.cam_ids[i], sc.width, sc.height, sc.K[i], sc.R[i], sc.t[i], sc.median_depth[i], sc.neighbors[i])
        A.add_image(*args, line3d.undistort_points(sc.segs[i], sc.K[i], lens))
        B.add_image(*args, sc.segs[i], lens=lens)
    for L in (A, B):
        L.match_images()
        L.reconstruct_3d_lines(3, True)
    a, b = A.lines(), B.lines()
    assert A.stats()["lines3D"] > 10
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k
    A.close()
    B.close()
