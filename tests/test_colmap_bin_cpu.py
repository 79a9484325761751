"""L3DPP::readColmap on COLMAP's binary model (cameras.bin / images.bin / points3D.bin) and on every lens model it reads, against an
independent writer of both formats (COLMAP's documented layouts, written here with struct.pack / text formatting)."""
import struct

import numpy as np
import pytest

from line3dpp_b200 import capi, line3d

NONE = 2 ** 64 - 1
# COLMAP model name -> (model_id, parameter names in COLMAP's order)
MODELS = {
    "SIMPLE_PINHOLE": (0, "f cx cy"), "PINHOLE": (1, "fx fy cx cy"), "SIMPLE_RADIAL": (2, "f cx cy k"), "RADIAL": (3, "f cx cy k1 k2"),
    "OPENCV": (4, "fx fy cx cy k1 k2 p1 p2"), "OPENCV_FISHEYE": (5, "fx fy cx cy k1 k2 k3 k4"),
    "FULL_OPENCV": (6, "fx fy cx cy k1 k2 p1 p2 k3 k4 k5 k6"), "FOV": (7, "fx fy cx cy omega"), "SIMPLE_RADIAL_FISHEYE": (8, "f cx cy k"),
    "RADIAL_FISHEYE": (9, "f cx cy k1 k2"), "THIN_PRISM_FISHEYE": (10, "fx fy cx cy k1 k2 p1 p2 k3 k4 sx1 sy1"),
}
FISHEYE = {"OPENCV_FISHEYE", "SIMPLE_RADIAL_FISHEYE", "RADIAL_FISHEYE"}
OLD_SIX = ["SIMPLE_PINHOLE", "PINHOLE", "SIMPLE_RADIAL", "RADIAL", "OPENCV", "FULL_OPENCV"]

CAMERAS = {   # camera_id: (model, width, height, params)
    1: ("SIMPLE_PINHOLE", 640, 480, [500.5, 320, 240]),
    2: ("PINHOLE", 640, 480, [500, 510, 321, 239]),
    3: ("SIMPLE_RADIAL", 640, 480, [400, 300, 200, 0.01]),
    4: ("RADIAL", 640, 480, [410, 310, 210, 0.02, -0.03]),
    5: ("OPENCV", 800, 600, [700, 710, 400, 300, 0.1, 0.2, 0.001, 0.002]),
    6: ("FULL_OPENCV", 800, 600, [701, 711, 401, 301, 0.11, 0.21, 0.0011, 0.0021, 0.31, 0.04, -0.05, 0.006]),
    7: ("OPENCV_FISHEYE", 1600, 1200, [600, 605, 800, 600, 0.05, -0.01, 0.003, -0.0005]),
    8: ("SIMPLE_RADIAL_FISHEYE", 1600, 1200, [620, 799.5, 600.5, 0.07]),
    9: ("RADIAL_FISHEYE", 1600, 1200, [630, 801, 599, 0.06, -0.02]),
}


def _scene(cam_ids, seed=1):
    """images (id, q, t, camera_id, name, [(x, y, point3D_id or NONE)]) and points {id: xyz}; one image has an unknown camera, images
    observe points more than once, some observations have no point and one observed point is missing from the point list"""
    rng = np.random.default_rng(seed)
    NP = 30
    pts = {int(j) * 3 + 1: rng.uniform(-1, 1, 3) for j in range(NP)}
    ids = sorted(pts)
    images = []
    for n, cam in enumerate(list(cam_ids) + [99]):
        q = rng.normal(size=4) * 1.3
        t = rng.uniform(-2, 2, 3)
        seen = [int(v) for v in rng.choice(ids, size=9, replace=False)]
        seen.insert(3, seen[1])                                   # a repeated observation
        obs = [(1.5 + j, 2.25 - j, NONE if j % 4 == 2 else p) for j, p in enumerate(seen)]
        images.append((20 + 3 * n, q, t, cam, f"img_{n:03d}.jpg", obs))
    del pts[ids[5]]                                               # observed (maybe), never defined: stays at the origin
    return images, pts


def write_text(folder, cameras, images, pts):
    f = lambda v: repr(float(v))
    L = ["# Camera list with one line of data per camera:"]
    L += [f"{cid} {m} {w} {h} " + " ".join(f(v) for v in prm) for cid, (m, w, h, prm) in cameras.items()]
    (folder / "cameras.txt").write_text("\n".join(L) + "\n")
    L = ["# Image list with two lines of data per image:", "#   IMAGE_ID, QW, QX, QY, QZ, TX, TY, TZ, CAMERA_ID, NAME"]
    for iid, q, t, cam, name, obs in images:
        L.append(f"{iid} " + " ".join(f(v) for v in q) + " " + " ".join(f(v) for v in t) + f" {cam} {name}")
        L.append(" ".join(f"{f(x)} {f(y)} {-1 if p == NONE else p}" for x, y, p in obs))
    (folder / "images.txt").write_text("\n".join(L) + "\n")
    L = ["# 3D point list with one line of data per point:"]
    L += [f"{pid} {f(X[0])} {f(X[1])} {f(X[2])} 10 20 30 0.5 " + " ".join(f"{iid} {k}" for k, iid in enumerate((20, 23))) for pid, X in pts.items()]
    (folder / "points3D.txt").write_text("\n".join(L) + "\n")


def bin_cameras(cameras, model_id=None):
    b = struct.pack("<Q", len(cameras))
    for cid, (m, w, h, prm) in cameras.items():
        b += struct.pack("<IiQQ", cid, MODELS[m][0] if model_id is None else model_id, w, h) + struct.pack(f"<{len(prm)}d", *prm)
    return b


def bin_images(images):
    b = struct.pack("<Q", len(images))
    for iid, q, t, cam, name, obs in images:
        b += struct.pack("<I4d3dI", iid, *q, *t, cam) + name.encode() + b"\0" + struct.pack("<Q", len(obs))
        for x, y, p in obs:
            b += struct.pack("<ddQ", x, y, p)
    return b


def bin_points(pts):
    b = struct.pack("<Q", len(pts))
    for pid, X in pts.items():
        track = [(20, 0), (23, 1)]
        b += struct.pack("<Q3d3BdQ", pid, *X, 10, 20, 30, 0.5, len(track)) + b"".join(struct.pack("<II", i, k) for i, k in track)
    return b


def write_bin(folder, cameras, images, pts):
    (folder / "cameras.bin").write_bytes(bin_cameras(cameras))
    (folder / "images.bin").write_bytes(bin_images(images))
    (folder / "points3D.bin").write_bytes(bin_points(pts))


def read(folder, lenses=True):
    """readColmap with or without lenses: (cameras as dicts, '') or (None, error)"""
    try:
        return line3d.read_colmap(folder, lenses), ""
    except capi.L3DError as e:
        return None, str(e)


def _bits(c):
    """every field of a camera dict as bytes"""
    out = [str(c["id"]).encode(), c["image"].encode(), np.float32(c["median_depth"]).tobytes(), np.asarray(c["worldpoints"], np.uint32).tobytes()]
    out += [np.asarray(c[k], np.float64).tobytes() for k in ("K", "R", "t", "C", "radial", "tangential")]
    if "lens" in c:
        out += [str(c["lens"]["model"]).encode(), c["lens"]["k"].tobytes(), c["lens"]["p"].tobytes()]
    return out


def _expected(cameras, images, pts):
    """what readColmap returns, computed here: kept images in order, K / radial / tangential of main_colmap.cpp, the lens, the
    worldpoints and the float median depth"""
    exp = []
    for iid, q, t, cam, name, obs in images:
        if cam not in cameras:
            continue
        m, w, h, prm = cameras[cam]
        v = dict(zip(MODELS[m][1].split(), prm))
        fx, fy = (v["f"], v["f"]) if "f" in v else (v["fx"], v["fy"])
        K = np.array([[fx, 0, v["cx"]], [0, fy, v["cy"]], [0, 0, 1.0]])
        g = lambda k: float(v.get(k, 0.0))
        if m in FISHEYE:
            radial, tang = [0.0] * 3, [0.0] * 2
            k = [g("k"), 0, 0, 0, 0, 0] if "k" in v else [g("k1"), g("k2"), g("k3"), g("k4"), 0, 0]
            lens = dict(model=1, k=k, p=[0.0, 0.0])
        else:
            k1 = g("k") if "k" in v else g("k1")
            radial, tang = [k1, g("k2"), g("k3")], [g("p1"), g("p2")]
            lens = dict(model=0, k=[k1, g("k2"), g("k3"), g("k4"), g("k5"), g("k6")], p=tang)
        qq = np.asarray(q) / np.linalg.norm(q)
        wps = [int(p) for _, _, p in obs if p != NONE]
        exp.append(dict(id=iid, image=name, K=K, radial=radial, tangential=tang, lens=lens, q=qq, t=t, wps=wps))
    return exp


def _check_against_expected(cams, exp, pts, with_lens):
    assert [c["id"] for c in cams] == [e["id"] for e in exp]
    for c, e in zip(cams, exp):
        assert c["image"] == e["image"] and np.array_equal(c["K"], e["K"])
        assert c["radial"].tolist() == e["radial"] and c["tangential"].tolist() == e["tangential"]
        assert c["worldpoints"].tolist() == e["wps"]
        np.testing.assert_allclose(c["t"], e["t"], rtol=0, atol=0)
        w, x, y, z = e["q"]
        R = np.array([[1 - 2 * y * y - 2 * z * z, 2 * x * y - 2 * z * w, 2 * x * z + 2 * y * w], [2 * x * y + 2 * z * w, 1 - 2 * x * x - 2 * z * z, 2 * y * z - 2 * x * w],
                      [2 * x * z - 2 * y * w, 2 * y * z + 2 * x * w, 1 - 2 * x * x - 2 * y * y]])
        np.testing.assert_allclose(c["R"], R, atol=1e-14)
        P = np.array([pts.get(p, np.zeros(3)) for p in e["wps"]])
        dep = np.sort(np.array([np.float32(np.linalg.norm(c["C"] - p)) for p in P], np.float32))
        assert c["median_depth"] == dep[len(dep) // 2]
        if with_lens:
            assert c["lens"]["model"] == e["lens"]["model"]
            assert c["lens"]["k"].tolist() == e["lens"]["k"] and c["lens"]["p"].tolist() == e["lens"]["p"]
        else:
            assert "lens" not in c


@pytest.fixture
def every_model(tmp_path):
    images, pts = _scene(CAMERAS)
    t, b, both = tmp_path / "txt", tmp_path / "bin", tmp_path / "both"
    for d in (t, b, both):
        d.mkdir()
    write_text(t, CAMERAS, images, pts)
    write_bin(b, CAMERAS, images, pts)
    write_text(both, CAMERAS, images, pts)
    (both / "cameras.bin").write_bytes(b"garbage")                # the text files win: the binary ones are not read
    return t, b, both, images, pts


def test_binary_equals_text_field_for_field(every_model):
    t, b, both, images, pts = every_model
    ct, e1 = read(t)
    cb, e2 = read(b)
    cboth, e3 = read(both)
    assert ct is not None and cb is not None and cboth is not None, (e1, e2, e3)
    assert len(ct) == len(CAMERAS) and len(ct) == len(cb)
    for a, c, d in zip(ct, cb, cboth):
        assert _bits(a) == _bits(c) == _bits(d)
    _check_against_expected(cb, _expected(CAMERAS, images, pts), pts, with_lens=True)


@pytest.mark.parametrize("fmt", ["txt", "bin"])
def test_old_models_read_as_before_with_or_without_lenses(tmp_path, fmt):
    cams6 = {cid: v for cid, v in CAMERAS.items() if v[0] in OLD_SIX}
    images, pts = _scene(cams6, seed=2)
    (write_text if fmt == "txt" else write_bin)(tmp_path, cams6, images, pts)
    plain, err = read(tmp_path, lenses=False)
    assert plain is not None, err
    lensed, err = read(tmp_path)
    assert lensed is not None, err
    exp = _expected(cams6, images, pts)
    _check_against_expected(plain, exp, pts, with_lens=False)
    _check_against_expected(lensed, exp, pts, with_lens=True)
    for a, c in zip(plain, lensed):
        assert _bits(a) == _bits({k: v for k, v in c.items() if k != "lens"})


@pytest.mark.parametrize("fmt", ["txt", "bin"])
def test_lens_contents_per_model(tmp_path, fmt):
    images, pts = _scene(CAMERAS, seed=3)
    (write_text if fmt == "txt" else write_bin)(tmp_path, CAMERAS, images, pts)
    cams, err = read(tmp_path)
    assert cams is not None, err
    by_cam = {im[0]: im[3] for im in images}
    seen = set()
    for c in cams:
        m, _, _, prm = CAMERAS[by_cam[c["id"]]]
        seen.add(m)
        lens = c["lens"]
        if m == "FULL_OPENCV":
            assert lens["model"] == 0 and lens["k"].tolist() == [prm[4], prm[5], prm[8], prm[9], prm[10], prm[11]] and lens["p"].tolist() == prm[6:8]
            assert c["radial"].tolist() == [prm[4], prm[5], prm[8]]          # k4..k6 reach the lens only
        elif m == "OPENCV_FISHEYE":
            assert lens["model"] == 1 and lens["k"].tolist() == prm[4:8] + [0, 0] and not lens["p"].any()
        elif m == "SIMPLE_RADIAL_FISHEYE":
            assert lens["model"] == 1 and lens["k"].tolist() == [prm[3], 0, 0, 0, 0, 0]
        elif m == "RADIAL_FISHEYE":
            assert lens["model"] == 1 and lens["k"].tolist() == [prm[3], prm[4], 0, 0, 0, 0]
        if m in FISHEYE:
            assert not c["radial"].any() and not c["tangential"].any()
    assert seen == {v[0] for v in CAMERAS.values()}


@pytest.mark.parametrize("fmt", ["txt", "bin"])
def test_rejections(tmp_path, fmt):
    write = write_text if fmt == "txt" else write_bin
    for model in sorted(FISHEYE):
        d = tmp_path / f"fe_{model}"
        d.mkdir()
        cams = {1: CAMERAS[1], 5: next(v for v in CAMERAS.values() if v[0] == model)}
        images, pts = _scene(cams, seed=4)
        write(d, cams, images, pts)
        bad, err = read(d, lenses=False)
        assert bad is None and "fisheye model " + model in err and "lenses" in err, err
        ok, err = read(d)
        assert ok is not None, err
    for model, prm in (("FOV", [500, 500, 320, 240, 0.9]), ("THIN_PRISM_FISHEYE", [500, 500, 320, 240] + [0.01] * 8)):
        d = tmp_path / f"rej_{model}"
        d.mkdir()
        cams = {1: CAMERAS[1], 3: (model, 640, 480, prm)}
        images, pts = _scene(cams, seed=5)
        write(d, cams, images, pts)
        for lenses in (False, True):
            bad, err = read(d, lenses)
            assert bad is None and f"camera model {model} unknown! (camera 3)" in err, err


def _small():
    cams = {4: CAMERAS[5]}
    images = [(7, [1, 0, 0, 0], [0.5, 0, 2], 4, "a.png", [(1.0, 2.0, 11), (3.0, 4.0, NONE)])]
    pts = {11: np.array([0.1, 0.2, 5.0])}
    return cams, images, pts


def malformed_binary_models():
    """a small binary model's files and every malformed variant of them: (good files, [(name, replaced files, check)]), where
    check(error) holds for the message readColmap must give"""
    cams, images, pts = _small()
    good = {"cameras.bin": bin_cameras(cams), "images.bin": bin_images(images), "points3D.bin": bin_points(pts)}
    out = []
    for name, data in good.items():
        for cut in range(len(data)):
            out.append((f"{name}_cut{cut}", {name: data[:cut]}, lambda e, name=name: name in e and ("truncated" in e or "exceeds" in e)))
    for name, data in good.items():                               # a count the file cannot hold: no allocation of that size
        out.append((f"{name}_count", {name: struct.pack("<Q", 2 ** 60) + data[8:]}, lambda e, name=name: name in e and "exceeds" in e))
    out.append(("cameras_40_bytes", {"cameras.bin": struct.pack("<Q", 2 ** 60) + b"\0" * 32}, lambda e: "cameras.bin" in e))
    name_at = 8 + 4 + 56 + 4
    out.append(("unterminated_name", {"images.bin": good["images.bin"][:name_at] + b"x" * 40},   # the name never ends
                lambda e: "images.bin" in e and "unterminated" in e))
    out.append(("model_42", {"cameras.bin": bin_cameras(cams, model_id=42)}, lambda e: "cameras.bin" in e and "42" in e and "unknown" in e))
    out.append(("model_-1", {"cameras.bin": bin_cameras(cams, model_id=-1)}, lambda e: "unknown" in e))
    big = [(7, [1, 0, 0, 0], [0.5, 0, 2], 4, "a.png", [(1.0, 2.0, 2 ** 33)])]
    out.append(("image_point_id", {"images.bin": bin_images(big)}, lambda e: "images.bin" in e and "unsigned int" in e))
    out.append(("point_id", {"points3D.bin": bin_points({2 ** 32: np.zeros(3)})}, lambda e: "points3D.bin" in e and "unsigned int" in e))
    return good, out


def write_files(d, good, replaced):
    for k, v in good.items():
        (d / k).write_bytes(replaced.get(k, v))


def test_malformed_binary_files_fail_cleanly(tmp_path):
    good, variants = malformed_binary_models()
    d = tmp_path / "m"
    d.mkdir()
    write_files(d, good, {})
    ok, err = read(d)
    assert ok is not None and len(ok) == 1 and ok[0]["worldpoints"].tolist() == [11], err
    for name, replaced, check in variants:
        write_files(d, good, replaced)
        bad, err = read(d)
        assert bad is None and check(err), (name, err)
    assert sum(1 for name, _, _ in variants if "_cut" in name) == sum(len(v) for v in good.values())
    write_files(d, good, {})
    (d / "points3D.bin").unlink()
    bad, err = read(d)
    assert bad is None and "does not exist" in err


def test_sfm_frontend_colmap_mode_reads_the_binary_model(tmp_path):
    """examples/sfm_frontend.cpp's colmap mode reads a binary model, reports every camera's lens model, and - like its other modes -
    stops with "no usable CUDA device" without a GPU (with one: it has no segments, so fewer than three images are usable)"""
    import os
    import subprocess
    from line3dpp_b200 import build
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    so = build.build()
    exe = tmp_path / "sfm_frontend"
    cmd = ["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", os.path.join(root, "examples", "sfm_frontend.cpp"), "-I" + os.path.join(root, "include"),
           "-L" + os.path.dirname(so), "-ll3d_b200", "-Wl,-rpath," + os.path.dirname(so), "-o", str(exe)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    model, segs = tmp_path / "sparse" / "0", tmp_path / "segs"
    model.mkdir(parents=True)
    segs.mkdir()
    images, pts = _scene(CAMERAS, seed=7)
    write_bin(model, CAMERAS, images, pts)
    r = subprocess.run([str(exe), "colmap", str(model), str(segs), str(tmp_path)], capture_output=True, text=True)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("camera ")]
    assert len(lines) == len(CAMERAS), r.stdout
    kinds = [ln.split(": ")[1].split(" lens")[0] for ln in lines]
    assert kinds == ["fisheye" if CAMERAS[im[3]][0] in FISHEYE else "radtan" for im in images if im[3] in CAMERAS]
    assert "k = 0.05 -0.01 0.003 -0.0005 0 0" in r.stdout                # OPENCV_FISHEYE's k1..k4
    try:
        import torch
        gpu = torch.cuda.is_available()
    except ImportError:
        gpu = False
    if gpu:
        assert r.returncode == 1 and "fewer than three usable images" in r.stderr, (r.returncode, r.stderr)
    else:
        assert r.returncode == 3 and "no usable CUDA device" in r.stderr, (r.returncode, r.stderr)
    r = subprocess.run([str(exe), "colmap", str(tmp_path / "nowhere"), str(segs), str(tmp_path)], capture_output=True, text=True)
    assert r.returncode == 1 and "does not exist" in r.stderr
