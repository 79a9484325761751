"""The readers of all six SfM formats and the frontend helpers without a GPU (include/line3d_io.h, csrc/line3d_sfm.cc, DESIGN.md §6b):
a synthetic model written in each format is read back exactly, malformed input is rejected with a message, and the reader file
alone survives every valid and malformed file under AddressSanitizer."""
import ctypes
import fnmatch
import gzip
import math
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from line3dpp_b200 import build, capi, line3d
from tests import sfm_scene as ss
from tests import test_colmap_bin_cpu as cb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def scene():
    return ss.Scene()


def _has_gpu():
    import torch
    return torch.cuda.is_available()


# ---------------------------------------------------------------------------------------------- helpers on Line3D
@pytest.mark.parametrize("rpy", [(0.0, 0.0, 0.0), (0.3, -0.7, 2.9), (-math.pi, math.pi / 2, -math.pi), (1e-9, -2.5, 0.125)])
def test_rotation_from_rpy_matches_restatement(rpy):
    R = line3d.rotation_from_rpy(*rpy)
    assert np.array_equal(R, ss.rotation_from_rpy(*rpy))
    np.testing.assert_allclose(R @ R.T, np.eye(3), atol=1e-15)
    r, p, y = rpy
    Rx = np.array([[1, 0, 0], [0, math.cos(r), -math.sin(r)], [0, math.sin(r), math.cos(r)]])
    Ry = np.array([[math.cos(p), 0, math.sin(p)], [0, 1, 0], [-math.sin(p), 0, math.cos(p)]])
    Rz = np.array([[math.cos(y), -math.sin(y), 0], [math.sin(y), math.cos(y), 0], [0, 0, 1]])
    np.testing.assert_allclose(R, Rz @ Ry @ Rx, atol=1e-15)


@pytest.mark.parametrize("signs", [(1, 1), (-1, 1), (1, -1), (-1, -1)])
def test_decompose_projection_matrix(signs):
    rng = np.random.default_rng(3 + signs[0] + 2 * signs[1])
    for _ in range(20):
        q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        R = q * np.sign(np.linalg.det(q))
        K = np.array([[signs[0] * rng.uniform(500, 3000), rng.uniform(-2, 2), rng.uniform(300, 1500)],
                      [0, signs[1] * rng.uniform(500, 3000), rng.uniform(300, 1000)], [0, 0, 1]])
        t = rng.uniform(-5, 5, 3)
        P = K @ np.hstack([R, t[:, None]]) * rng.uniform(0.5, 2.0)       # any scale: K is normalised to K(2,2) = 1
        Kd, Rd, td = line3d.decompose_projection_matrix(P)
        Kr, Rr, tr = ss.decompose_restated(P)
        np.testing.assert_allclose(Kd, Kr, rtol=1e-12, atol=1e-9); np.testing.assert_allclose(Rd, Rr, atol=1e-12); np.testing.assert_allclose(td, tr, atol=1e-12)
        assert abs(Kd[2, 2] - 1.0) < 1e-15 and (np.diag(Kd) > 0).all() and abs(Kd[1, 0]) + abs(Kd[2, 0]) + abs(Kd[2, 1]) < 1e-9
        # the decomposition reproduces P up to its scale; with positive focal signs it is K, R, t themselves
        np.testing.assert_allclose(Kd @ np.hstack([Rd, td[:, None]]), P / (P[2, :3] @ Rd[2]), rtol=1e-12, atol=1e-9)
        if signs == (1, 1):
            np.testing.assert_allclose(Kd, K, rtol=1e-12, atol=1e-9); np.testing.assert_allclose(Rd, R, atol=1e-12)
            np.testing.assert_allclose(td, t, atol=1e-12 * 5)


def test_sequential_neighbors():
    def ref(i, n, k):                                 # main_mavmap.cpp:312-321
        out = []
        for j in range(i - 1, -1, -1):
            if len(out) >= k // 2:
                break
            out.append(j)
        for j in range(i + 1, n):
            if len(out) >= k:
                break
            out.append(j)
        return out
    for k in (2, 3, 10):
        for n in (1, 2, 5, 12, 30):
            for i in sorted({0, 1, n // 2, n - 2, n - 1} - {-1}):
                if 0 <= i < n:
                    assert line3d.sequential_neighbors(i, n, k) == ref(i, n, k), (i, n, k)
    assert line3d.sequential_neighbors(0, 30, 10) == list(range(1, 11))
    assert line3d.sequential_neighbors(29, 30, 10) == [28, 27, 26, 25, 24]
    assert line3d.sequential_neighbors(15, 30, 3) == [14, 16, 17]


# ---------------------------------------------------------------------------------------------- readers
def test_mavmap_reader(scene, tmp_path):
    p = tmp_path / "mavmap.txt"
    scene.write_mavmap(p, tail="short line ends the list\nimg99, this camera is never read, 0, 0, 0, 0, 0, 0, 0, 0, 0,\n")
    cams = line3d.read_mavmap(p)
    assert [c["id"] for c in cams] == list(range(scene.V)) and [c["image"] for c in cams] == [f"img{i}" for i in range(scene.V)]
    for i, c in enumerate(cams):
        np.testing.assert_allclose(c["K"], scene.K[i], rtol=0, atol=1e-12)
        np.testing.assert_allclose(c["R"], scene.R_mav[i], rtol=0, atol=1e-12)
        np.testing.assert_allclose(c["t"], scene.t_mav[i], rtol=0, atol=1e-12)
        np.testing.assert_allclose(c["C"], scene.C[i], rtol=0, atol=1e-12)
        assert np.array_equal(c["R"], scene.R_mav[i]) and np.array_equal(c["t"], scene.t_mav[i])
        assert not c["radial"].any() and not c["tangential"].any() and c["median_depth"] == 0 and len(c["worldpoints"]) == 0


def test_openmvg_reader(scene, tmp_path):
    p = tmp_path / "sfm_data.json"
    p.write_text(scene.openmvg_text())
    cams = line3d.read_openmvg(p)
    exp = scene.openmvg_expected()
    keep = [i for i in range(scene.V) if exp[i][1] is not None]
    assert [c["id"] for c in cams] == [100 + i for i in keep] and len(keep) >= 6
    for c, i in zip(cams, keep):
        assert c["image"] == f"img{i}.jpg"
        assert np.array_equal(c["K"], np.array([[scene.K[i][0, 0], 0, scene.K[i][0, 2]], [0, scene.K[i][0, 0], scene.K[i][1, 2]], [0, 0, 1]]))
        assert np.array_equal(c["R"], scene.R[i]) and np.array_equal(c["t"], scene.t[i]) and np.array_equal(c["C"], scene.C[i])
        r, t = scene.openmvg_distortion(i)
        assert np.array_equal(c["radial"], r) and np.array_equal(c["tangential"], t), (i, scene.MODELS[i % 6])
        assert c["worldpoints"].tolist() == exp[i][0] and c["median_depth"] == exp[i][1]


def test_openmvg_reader_first_entry_without_model_name(scene, tmp_path):
    """no polymorphic_name before any named entry: the reference's cam_model is still empty, so there is no distortion"""
    import json
    doc = json.loads(scene.openmvg_text())
    del doc["intrinsics"][0]["value"]["polymorphic_name"]
    p = tmp_path / "sfm_data.json"
    p.write_text(json.dumps(doc))
    c = line3d.read_openmvg(p)[0]
    assert not c["radial"].any() and not c["tangential"].any()


def test_pix4d_reader_needs_a_gpu(scene, tmp_path):
    if _has_gpu():
        pytest.skip("a GPU is present (tests/test_sfm_gpu.py)")
    scene.write_pix4d(tmp_path)
    with pytest.raises(capi.L3DError, match="no usable CUDA device"):
        line3d.read_pix4d(tmp_path, "proj")


# ---------------------------------------------------------------------------------------------- NVM, Bundler, COLMAP text
def write_nvm(path):
    """a synthetic NVM_V3 model: (q, C, f, d, pts, vis) as written"""
    rng = np.random.default_rng(3)
    V, NP = 5, 40
    q = rng.normal(size=(V, 4)); q /= np.linalg.norm(q, axis=1, keepdims=True)
    Cc = rng.uniform(-3, 3, (V, 3)); f = rng.uniform(800, 2500, V); d = np.array([0, 0.01, 0, -0.02, 0])
    pts = rng.uniform(-1, 1, (NP, 3))
    vis = [sorted(rng.choice(V, size=rng.integers(2, V + 1), replace=False).tolist()) for _ in range(NP)]
    lines = ["NVM_V3", "", str(V)]
    for i in range(V):
        lines.append(f"dir/img{i}.jpg\t{f[i]:.10f} {q[i,0]:.12f} {q[i,1]:.12f} {q[i,2]:.12f} {q[i,3]:.12f} {Cc[i,0]:.12f} {Cc[i,1]:.12f} {Cc[i,2]:.12f} {d[i]:.6f} 0")
    lines += ["", str(NP)]
    for j in range(NP):
        meas = " ".join(f"{c} {7 * j + c} {10.5 + c} {-3.25 + j}" for c in vis[j])
        lines.append(f"{pts[j,0]:.12f} {pts[j,1]:.12f} {pts[j,2]:.12f} 255 128 0 {len(vis[j])} {meas}")
    path.write_text("\n".join(lines) + "\n0\n")
    return q, Cc, f, d, pts, vis


def test_nvm_reader_round_trip(tmp_path):
    """L3DPP::readNVM (include/line3d_io.h; restates main_vsfm.cpp:143-310) on a synthetic NVM_V3 model"""
    path = tmp_path / "model.nvm"
    q, Cc, f, d, pts, vis = write_nvm(path)
    V, NP = len(q), len(pts)
    cams = line3d.read_nvm(path)
    assert len(cams) == V
    for i, c in enumerate(cams):
        qw, qx, qy, qz = [float(f"{v:.12f}") for v in q[i]]
        R = np.array([[1 - 2 * qy * qy - 2 * qz * qz, 2 * qx * qy - 2 * qz * qw, 2 * qx * qz + 2 * qy * qw],
                      [2 * qx * qy + 2 * qz * qw, 1 - 2 * qx * qx - 2 * qz * qz, 2 * qy * qz - 2 * qx * qw],
                      [2 * qx * qz - 2 * qy * qw, 2 * qy * qz + 2 * qx * qw, 1 - 2 * qx * qx - 2 * qy * qy]])
        Ci = np.array([float(f"{v:.12f}") for v in Cc[i]])
        np.testing.assert_allclose(c["R"], R, atol=1e-14)
        np.testing.assert_allclose(c["t"], -R @ Ci, atol=1e-13)
        assert c["image"] == f"dir/img{i}.jpg" and abs(c["focal"] - np.float32(f[i])) < 1e-3 and abs(c["distortion"] - d[i]) < 1e-7
        mine = [j for j in range(NP) if i in vis[j]]
        assert c["worldpoints"].tolist() == mine
        dep = np.sort(np.array([np.float32(np.linalg.norm(np.array([float(f"{v:.12f}") for v in pts[j]]) - Ci)) for j in mine], np.float32))
        assert c["median_depth"] == (dep[len(dep) // 2] if len(dep) else 0.0)
    with pytest.raises(capi.L3DError, match="cannot open"):
        line3d.read_nvm(tmp_path / "missing.nvm")
    (tmp_path / "empty.nvm").write_text("NVM_V3\n\n0\n")
    with pytest.raises(capi.L3DError, match="No aligned cameras"):
        line3d.read_nvm(tmp_path / "empty.nvm")


def test_nvm_reader_on_the_reference_test_data(tmp_path):
    """readNVM on the reference's own testdata/vsfm_result.nvm (every camera, the first 4500 points: tests/golden/vsfm_result_head.nvm.gz)
    equals the committed inputs of the nvm configuration (cameras) and the numpy reader of tests/golden/make_nvm_inputs.py
    (world-point lists, median depths)"""
    path = tmp_path / "vsfm_result.nvm"
    path.write_bytes(gzip.decompress(open(os.path.join(ROOT, "tests", "golden", "vsfm_result_head.nvm.gz"), "rb").read()))
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from make_nvm_inputs import read_nvm
    from tests import nvm_util as nu
    inp = nu.load_inputs()
    _, wps, depths = read_nvm(path)
    cams = line3d.read_nvm(path)
    assert len(cams) == inp["V"]
    L = capi.lib()
    for i, c in enumerate(cams):
        np.testing.assert_allclose(c["R"], inp["R"][i], atol=1e-15)
        np.testing.assert_allclose(c["t"], inp["t"][i], atol=1e-13)
        d = np.sort(np.array(depths[i], np.float32))
        assert len(d) > 0 and c["median_depth"] == d[len(d) // 2] and np.array_equal(c["worldpoints"], np.array(wps[i], np.uint32))
        K = np.zeros(9)
        L.l3dpp_intrinsics_from_focal(ctypes.c_float(c["focal"]), int(inp["wh"][i][0]), int(inp["wh"][i][1]), K.ctypes.data_as(ctypes.c_void_p))
        assert np.array_equal(K.reshape(3, 3), inp["K"][i])
    assert sum(len(c["worldpoints"]) for c in cams) > 10000


NVM_CAMERA = "img0.jpg 1000 1 0 0 0 0 0 0 0 0\n"
# (name, text, message): a truncated camera section is an error, not a default camera; a count the file does not hold allocates nothing
BAD_NVM = [("empty", "NVM_V3\n\n0\n", "No aligned cameras"),
           ("short_camera_line", "NVM_V3\n\n3\n" + NVM_CAMERA + "img1.jpg 1000 1 0 0 0\n", "camera"),
           ("truncated_camera_list", "NVM_V3\n\n2\n" + NVM_CAMERA, "end of file"),
           ("huge_camera_count", "NVM_V3\n\n4294967295\n" + NVM_CAMERA, "end of file in the camera list"),
           ("unknown_camera", "NVM_V3\n\n1\n" + NVM_CAMERA + "\n1\n0 0 1 255 0 0 1 7 0 1.5 2.5\n", "malformed measurement list")]


def test_nvm_reader_rejects_truncated_camera_list(tmp_path):
    for name, text, msg in BAD_NVM:
        f = tmp_path / f"{name}.nvm"
        f.write_text(text)
        with pytest.raises(capi.L3DError) as e:
            line3d.read_nvm(f)
        assert msg in str(e.value), (name, str(e.value))


def _rot(rng):
    q = rng.normal(size=4); q /= np.linalg.norm(q)
    w, x, y, z = q
    return q, np.array([[1 - 2 * y * y - 2 * z * z, 2 * x * y - 2 * z * w, 2 * x * z + 2 * y * w], [2 * x * y + 2 * z * w, 1 - 2 * x * x - 2 * z * z, 2 * y * z - 2 * x * w],
                        [2 * x * z - 2 * y * w, 2 * y * z + 2 * x * w, 1 - 2 * x * x - 2 * y * y]])


def write_bundler(folder):
    """a synthetic bundle.rd.out and image list in folder: (R, t, f, k, pts, vis) as written"""
    rng = np.random.default_rng(5)
    V, NP = 4, 30
    Rs = [_rot(rng)[1] for _ in range(V)]; ts = rng.uniform(-2, 2, (V, 3)); f = rng.uniform(500, 2000, V); k = rng.uniform(-0.1, 0.1, (V, 2))
    pts = rng.uniform(-1, 1, (NP, 3))
    vis = [sorted(rng.choice(V, size=rng.integers(2, V + 1), replace=False).tolist()) for _ in range(NP)]
    L = ["# Bundle file v0.3", f"{V} {NP}"]
    for i in range(V):
        L.append(f"{f[i]:.10f} {k[i,0]:.10f} {k[i,1]:.10f}")
        L += [" ".join(f"{v:.12f}" for v in Rs[i][r]) for r in range(3)]
        L.append(" ".join(f"{v:.12f}" for v in ts[i]))
    for j in range(NP):
        L += [" ".join(f"{v:.12f}" for v in pts[j]), "255 0 0", f"{len(vis[j])} " + " ".join(f"{c} {j} 1.5 -2.5" for c in vis[j])]
    (folder / "bundle.rd.out").write_text("\n".join(L) + "\n")
    (folder / "list.txt").write_text("a.jpg 0 123\nb.jpg\n\nd.jpg 1 2\n")
    return Rs, ts, f, k, pts, vis


BUNDLER_CAMERA = "1000 0 0\n1 0 0\n0 1 0\n0 0 1\n0 0 0\n"
BAD_BUNDLER = [("empty", "# Bundle file v0.3\n0 0\n", "No cameras"),
               ("huge_camera_count", "# Bundle file v0.3\n4294967295 1\n" + BUNDLER_CAMERA, "truncated or malformed camera 1 "),
               ("unknown_camera", "# Bundle file v0.3\n1 1\n" + BUNDLER_CAMERA + "0 0 1\n255 0 0\n1 5 0 1.5 2.5\n", "malformed view list")]


def test_bundler_reader(tmp_path):
    """L3DPP::readBundler (include/line3d_io.h; restates main_bundler.cpp:143-286) on a synthetic bundle.rd.out"""
    Rs, ts, f, k, pts, vis = write_bundler(tmp_path)
    V, NP = len(Rs), len(pts)
    cams = line3d.read_bundler(tmp_path / "bundle.rd.out", tmp_path / "list.txt")
    assert len(cams) == V
    rd = lambda a: np.array([float(f"{v:.12f}") for v in np.ravel(a)]).reshape(np.shape(a))
    for i, c in enumerate(cams):
        R = rd(Rs[i]); R[1:] *= -1
        t = rd(ts[i]); t[1:] *= -1
        np.testing.assert_allclose(c["R"], R, atol=1e-15); np.testing.assert_allclose(c["t"], t, atol=1e-15)
        Ci = -R.T @ t
        np.testing.assert_allclose(c["C"], Ci, atol=1e-14)
        assert c["id"] == i and not c["has_K"] and abs(c["focal"] - np.float32(float(f"{f[i]:.10f}"))) < 1e-3
        np.testing.assert_allclose(c["radial"][:2], np.float32(rd(k[i])), atol=1e-9); assert not c["radial"][2:].any() and not c["tangential"].any()
        mine = [j for j in range(NP) if i in vis[j]]
        assert c["worldpoints"].tolist() == mine
        dep = np.sort(np.array([np.float32(np.linalg.norm(rd(pts[j]) - c["C"])) for j in mine], np.float32))
        assert c["median_depth"] == (dep[len(dep) // 2] if len(dep) else np.float32(0))
    assert [c["image"] for c in cams] == ["a.jpg", "b.jpg", "", "d.jpg"]
    for name, text, msg in BAD_BUNDLER:
        (tmp_path / name).write_text(text)
        with pytest.raises(capi.L3DError) as e:
            line3d.read_bundler(tmp_path / name)
        assert msg in str(e.value), (name, str(e.value))


def write_colmap_text(folder):
    """a synthetic COLMAP text model in folder: [(image id, camera id, q, t, world points)] and the points as written"""
    rng = np.random.default_rng(6)
    cam_lines = ["# Camera list", "1 SIMPLE_PINHOLE 640 480 500.5 320 240", "2 PINHOLE 640 480 500 510 321 239", "3 SIMPLE_RADIAL 640 480 400 300 200 0.01",
                 "4 RADIAL 640 480 410 310 210 0.02 -0.03", "5 OPENCV 800 600 700 710 400 300 0.1 0.2 0.001 0.002",
                 "6 FULL_OPENCV 800 600 701 711 401 301 0.11 0.21 0.0011 0.0021 0.31 0 0 0"]
    (folder / "cameras.txt").write_text("\n".join(cam_lines) + "\n")
    NP = 25
    pts = rng.uniform(-1, 1, (NP, 3))
    imgs, L = [], ["# Image list with two lines of data per image:"]
    for n, (img_id, cam_id) in enumerate([(10, 1), (11, 2), (12, 3), (13, 4), (14, 5), (15, 6), (16, 99)]):
        q, R = _rot(rng)
        q = q * 1.7                                   # rotationFromQ normalises (line3D.cc:2737-2754)
        t = rng.uniform(-2, 2, 3)
        seen = sorted(rng.choice(NP, size=8, replace=False).tolist())
        obs = " ".join(f"{1.0 + j} {2.0 + j} {(-1 if k % 3 == 0 else p)}" for k, (j, p) in enumerate(zip(range(8), seen)))
        L += [f"{img_id} {q[0]:.12f} {q[1]:.12f} {q[2]:.12f} {q[3]:.12f} {t[0]:.12f} {t[1]:.12f} {t[2]:.12f} {cam_id} im{img_id}.png", obs]
        imgs.append((img_id, cam_id, q, t, [p for k, p in enumerate(seen) if k % 3 != 0]))
    (folder / "images.txt").write_text("\n".join(L) + "\n")
    (folder / "points3D.txt").write_text("# 3D point list\n" + "\n".join(f"{j} {pts[j,0]:.12f} {pts[j,1]:.12f} {pts[j,2]:.12f} 1 2 3 0.5 10 1" for j in range(NP) if j != 7) + "\n")
    return imgs, pts


def test_colmap_reader(tmp_path):
    """L3DPP::readColmap (include/line3d_io.h; restates main_colmap.cpp:140-401) on a synthetic text model"""
    imgs, pts = write_colmap_text(tmp_path)
    cams = line3d.read_colmap(tmp_path, lenses=False)
    assert [c["id"] for c in cams] == [10, 11, 12, 13, 14, 15]                     # image 16 uses an unknown camera: dropped
    expK = {1: (500.5, 500.5, 320, 240), 2: (500, 510, 321, 239), 3: (400, 400, 300, 200), 4: (410, 410, 310, 210), 5: (700, 710, 400, 300), 6: (701, 711, 401, 301)}
    expD = {1: (0, 0, 0, 0, 0), 2: (0, 0, 0, 0, 0), 3: (0.01, 0, 0, 0, 0), 4: (0.02, -0.03, 0, 0, 0), 5: (0.1, 0.2, 0, 0.001, 0.002), 6: (0.11, 0.21, 0.31, 0.0011, 0.0021)}
    rd = lambda a: np.array([float(f"{v:.12f}") for v in np.ravel(a)])
    for c, (img_id, cam_id, q, t, seen) in zip(cams, imgs):
        fx, fy, cx, cy = expK[cam_id]
        assert np.array_equal(c["K"], np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1.0]])) and c["has_K"]
        np.testing.assert_allclose(np.concatenate([c["radial"], c["tangential"]]), expD[cam_id], atol=1e-15)
        qq = rd(q); qq = qq / np.linalg.norm(qq); w, x, y, z = qq
        R = np.array([[1 - 2 * y * y - 2 * z * z, 2 * x * y - 2 * z * w, 2 * x * z + 2 * y * w], [2 * x * y + 2 * z * w, 1 - 2 * x * x - 2 * z * z, 2 * y * z - 2 * x * w],
                      [2 * x * z - 2 * y * w, 2 * y * z + 2 * x * w, 1 - 2 * x * x - 2 * y * y]])
        np.testing.assert_allclose(c["R"], R, atol=1e-14); np.testing.assert_allclose(c["t"], rd(t), atol=1e-15)
        np.testing.assert_allclose(c["C"], -R.T @ rd(t), atol=1e-13)
        assert c["worldpoints"].tolist() == seen and c["image"] == f"im{img_id}.png"
        P = np.array([rd(pts[j]) if j != 7 else np.zeros(3) for j in seen])       # a point missing from points3D.txt stays at the origin
        dep = np.sort(np.array([np.float32(np.linalg.norm(c["C"] - p)) for p in P], np.float32))
        assert c["median_depth"] == dep[len(dep) // 2]
    with pytest.raises(capi.L3DError, match="does not exist"):
        line3d.read_colmap(tmp_path / "nowhere", lenses=False)
    (tmp_path / "cameras.txt").write_text("1 FISHEYE 10 10 1 2 3\n")
    with pytest.raises(capi.L3DError, match="FISHEYE unknown"):
        line3d.read_colmap(tmp_path, lenses=False)


# ---------------------------------------------------------------------------------------------- malformed input
def bad_mavmap(scene, tmp):
    p = tmp / "good_mavmap.txt"
    scene.write_mavmap(p)
    lines = p.read_text().split("\n")
    first = lines[2]
    out = [("truncated", lines[:2] + [", ".join(first.split(", ")[:6])], "truncated camera line (6 of 17 fields)"),
           ("non_numeric", lines[:2] + [first.replace(first.split()[1], "abc,", 1)], "non-numeric field 2"),
           ("model", lines[:2] + [first.replace("PINHOLE,", "OPENCV,")], "only PINHOLE"),
           ("empty", ["# only a comment"], "no camera")]
    return [(n, "\n".join(l) + "\n", m) for n, l, m in out]


def test_malformed_mavmap(scene, tmp_path):
    for name, text, msg in bad_mavmap(scene, tmp_path):
        p = tmp_path / f"{name}.txt"
        p.write_text(text)
        with pytest.raises(capi.L3DError) as e:
            line3d.read_mavmap(p)
        assert msg in str(e.value) and str(p) in str(e.value), (name, str(e.value))


def bad_openmvg(scene):
    import json
    good = scene.openmvg_text()
    doc = lambda: json.loads(good)
    out = []
    d = doc(); del d["views"][1]["value"]["ptr_wrapper"]["data"]["id_pose"]; out.append(("missing_key", json.dumps(d), "views[1].value.ptr_wrapper.data.id_pose: missing"))
    d = doc(); d["views"][0]["value"]["ptr_wrapper"]["data"]["id_view"] = "3"; out.append(("string_for_uint", json.dumps(d), "id_view: expected an unsigned integer"))
    d = doc(); d["views"][0]["value"]["ptr_wrapper"]["data"]["id_view"] = 4294967296; out.append(("uint_too_large", json.dumps(d), "out of range"))
    d = doc(); d["views"][0]["value"]["ptr_wrapper"]["data"]["id_view"] = 1.5; out.append(("fraction_for_uint", json.dumps(d), "expected an unsigned integer"))
    d = doc(); d["views"][0]["value"]["ptr_wrapper"]["data"]["id_view"] = -1; out.append(("negative_uint", json.dumps(d), "expected an unsigned integer"))
    d = doc(); d["structure"] = {}; out.append(("object_for_array", json.dumps(d), "structure: expected an array"))
    d = doc(); d["extrinsics"][0]["value"]["rotation"][2] = [1, 2]; out.append(("short_row", json.dumps(d), "extrinsics[0].value.rotation[2][2]: missing"))
    d = doc(); d["intrinsics"][2]["value"]["ptr_wrapper"]["data"]["disto_t2"] = [0, 0, 0, 0]; out.append(("short_disto", json.dumps(d), "disto_t2[4]: missing"))
    d = doc(); d["structure"][0]["value"]["X"][1] = None; out.append(("null_for_number", json.dumps(d), "X[1]: expected a number"))
    d = doc(); d["views"] = []; out.append(("no_views", json.dumps(d), "No aligned cameras"))
    out.append(("unterminated_string", good[:good.index('"img3.jpg"') + 5], "unterminated string"))
    out.append(("truncated", good[: len(good) // 2], "unexpected end"))
    out.append(("deep", "[" * 100000 + "]" * 100000, "nesting deeper than 64"))
    out.append(("trailing", good + " x", "text after the JSON document"))
    out.append(("bad_escape", good.replace('"img2.jpg"', '"img\\q.jpg"'), "bad escape"))
    out.append(("bad_unicode", good.replace('"img2.jpg"', '"img\\ud800.jpg"'), "unpaired surrogate"))
    out.append(("bad_number", good.replace('"width": 3072', '"width": 01', 1), "expected ',' or '}'"))
    out.append(("not_json", "\x00\x01garbage", "unexpected character"))
    return out


def test_malformed_openmvg(scene, tmp_path):
    for name, text, msg in bad_openmvg(scene):
        p = tmp_path / f"{name}.json"
        p.write_text(text)
        with pytest.raises(capi.L3DError) as e:
            line3d.read_openmvg(p)
        assert msg in str(e.value) and str(p) in str(e.value), (name, str(e.value))
    with pytest.raises(capi.L3DError, match="cannot open"):
        line3d.read_openmvg(tmp_path / "missing.json")


def bad_pix4d(scene, tmp):
    """(name, folder) pairs of projects the reader rejects while parsing (before the GPU step)"""
    out = []
    for name, edit, msg in (("truncated_block", lambda c, t: ("\n".join(c.split("\n")[:3 + 12 + 5]) + "\n", t), "is truncated"),
                            ("non_numeric_K", lambda c, t: (c.replace("\n0 0 1\n", "\n0 zero 1\n", 1), t), "expected 3 numbers (K row)"),
                            ("short_R_row", lambda c, t: (c.replace(c.split("\n")[3 + 9], "0.5 0.25"), t), "expected 3 numbers (R row)"),
                            ("non_numeric_xy", lambda c, t: (c, t.replace(" 2.5\n", "\n").replace("\n1000 ", "\n1000 x", 1)), "non-numeric image coordinates"),
                            ("obs_before_key", lambda c, t: (c, "1000 1.5 2.5 1\n" + t), "observation before the first key image")):
        d = tmp / name
        scene.write_pix4d(d)
        cf, tf = d / "proj_calibrated_camera_parameters.txt", d / "proj_tp_pix4d.txt"
        c, t = edit(cf.read_text(), tf.read_text())
        cf.write_text(c); tf.write_text(t)
        out.append((name, d, msg))
    return out


def test_malformed_pix4d(scene, tmp_path):
    for name, d, msg in bad_pix4d(scene, tmp_path):
        with pytest.raises(capi.L3DError) as e:
            line3d.read_pix4d(d, "proj")
        assert msg in str(e.value), (name, str(e.value))
    with pytest.raises(capi.L3DError, match="does not exist"):
        line3d.read_pix4d(tmp_path / "nowhere", "proj")


ASAN_DRIVER = r"""
#include "line3d_io.h"
#include "l3d_capi.h"
#include <cstdio>
// the reader file alone: the device entries readPix4D calls are stand-ins that report no device
extern "C" {
int l3d_ctx_create(int, l3d_ctx** out) { *out = nullptr; return L3D_ERR_CUDA; }
void l3d_ctx_destroy(l3d_ctx*) {}
const char* l3d_last_error(const l3d_ctx*) { return "no device"; }
int l3d_triangulate_points(l3d_ctx*, long long, const int64_t*, const int32_t*, const double*, int, const double*, double*, int32_t*, int) { return L3D_ERR_CUDA; }
int l3d_median_depths(l3d_ctx*, int, const int64_t*, const int32_t*, long long, const double*, const int32_t*, const double*, int32_t*, float*, int) { return L3D_ERR_CUDA; }
}
// argv: N <file> (NVM), B <file> (Bundler), C / L <folder> (COLMAP without / with lenses), M <file> (mavmap), O <file> (OpenMVG),
// P <folder> (Pix4D, prefix "proj"); prints "ok|err <cameras> <error empty>" per input
int main(int argc, char** argv)
{
    for (int i = 1; i + 1 < argc; i += 2) {
        std::string err;
        std::vector<L3DPP::SfMCamera> v;
        std::vector<L3DPP::NVMCamera> nv;
        std::vector<L3DPP::LensDistortion> lenses;
        const std::string path = argv[i + 1];
        bool ok;
        switch (argv[i][0]) {
        case 'N': ok = L3DPP::readNVM(path, nv, &err); break;
        case 'B': ok = L3DPP::readBundler(path, "", v, &err); break;
        case 'C': ok = L3DPP::readColmap(path, v, &err); break;
        case 'L': ok = L3DPP::readColmap(path, v, &err, &lenses); break;
        case 'M': ok = L3DPP::readMavmap(path, v, &err); break;
        case 'O': ok = L3DPP::readOpenMVG(path, v, &err); break;
        default: ok = L3DPP::readPix4D(path, "proj", v, &err);
        }
        std::printf("%s %zu %d\n", ok ? "ok" : "err", v.size() + nv.size(), (int)err.empty());
    }
    return 0;
}
"""


def test_readers_under_address_sanitizer(scene, tmp_path):
    """csrc/line3d_sfm.cc alone, built with ASan + UBSan, on valid and every malformed input of the six formats, COLMAP's binary
    files cut at every byte among them; allocations above 64 MB count as errors.  The Pix4D projects stop at the (stand-in) device
    step or earlier.  The NVM, Bundler and COLMAP readers may leave the cameras read before an error in their output."""
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no g++")
    drv = tmp_path / "drv.cc"
    drv.write_text(ASAN_DRIVER)
    exe = tmp_path / "drv"
    cmd = [gxx, "-std=c++17", "-g", "-O1", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "line3dpp_b200", "csrc", "line3d_sfm.cc"), str(drv), "-o", str(exe)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        if "sanitize" in r.stderr or "asan" in r.stderr:
            pytest.skip("this compiler cannot build with AddressSanitizer: " + r.stderr[-300:])
        raise AssertionError(r.stderr)
    args, expect = [], []
    scene.write_mavmap(tmp_path / "m.txt"); (tmp_path / "o.json").write_text(scene.openmvg_text()); scene.write_pix4d(tmp_path / "p")
    args += ["M", str(tmp_path / "m.txt"), "O", str(tmp_path / "o.json"), "P", str(tmp_path / "p")]
    expect += [f"ok {scene.V} 1", f"ok {sum(1 for e in scene.openmvg_expected() if e[1] is not None)} 1", "err 0 0"]
    for name, text, _ in bad_mavmap(scene, tmp_path):
        (tmp_path / f"bm_{name}").write_text(text); args += ["M", str(tmp_path / f"bm_{name}")]; expect.append("err 0 0")
    for name, text, _ in bad_openmvg(scene):
        (tmp_path / f"bo_{name}").write_text(text); args += ["O", str(tmp_path / f"bo_{name}")]; expect.append("err 0 0")
    for name, d, _ in bad_pix4d(scene, tmp_path):
        args += ["P", str(d)]; expect.append("err 0 0")

    def put(kind, path, n):                          # n cameras, or None: an error
        args.extend([kind, str(path)]); expect.append(f"ok {n} 1" if n is not None else "err * 0")
    write_nvm(tmp_path / "n.nvm"); put("N", tmp_path / "n.nvm", 5)
    head = gzip.decompress(open(os.path.join(ROOT, "tests", "golden", "vsfm_result_head.nvm.gz"), "rb").read())
    (tmp_path / "vsfm.nvm").write_bytes(head); put("N", tmp_path / "vsfm.nvm", int(head.split(b"\n")[2]))
    for name, text, _ in BAD_NVM:
        (tmp_path / f"bn_{name}").write_text(text); put("N", tmp_path / f"bn_{name}", None)
    (tmp_path / "b").mkdir(); write_bundler(tmp_path / "b"); put("B", tmp_path / "b" / "bundle.rd.out", 4)
    for name, text, _ in BAD_BUNDLER:
        (tmp_path / f"bb_{name}").write_text(text); put("B", tmp_path / f"bb_{name}", None)
    (tmp_path / "ct").mkdir(); write_colmap_text(tmp_path / "ct"); put("C", tmp_path / "ct", 6); put("L", tmp_path / "ct", 6)
    (tmp_path / "cf").mkdir(); (tmp_path / "cf" / "cameras.txt").write_text("1 FISHEYE 10 10 1 2 3\n")
    (tmp_path / "cf" / "images.txt").write_text(""); (tmp_path / "cf" / "points3D.txt").write_text(""); put("C", tmp_path / "cf", None)
    images, pts = cb._scene(cb.CAMERAS)
    for fmt, write in (("txt", cb.write_text), ("bin", cb.write_bin)):
        d = tmp_path / f"every_{fmt}"
        d.mkdir(); write(d, cb.CAMERAS, images, pts)
        put("L", d, len(cb.CAMERAS)); put("C", d, None)       # fisheye cameras need the lenses
    good, variants = cb.malformed_binary_models()
    for name, replaced in [("good", {})] + [(n, r) for n, r, _ in variants]:
        d = tmp_path / f"cbin_{name}"
        d.mkdir(); cb.write_files(d, good, replaced); put("L", d, 1 if name == "good" else None)
    env = dict(os.environ, ASAN_OPTIONS="max_allocation_size_mb=64:allocator_may_return_null=0:detect_leaks=1")
    r = subprocess.run([str(exe)] + args, capture_output=True, text=True, env=env)
    assert r.returncode == 0 and "Sanitizer" not in r.stderr, r.stderr[-2000:]
    got = r.stdout.split("\n")[:-1]
    assert len(got) == len(expect) and all(fnmatch.fnmatchcase(g, e) for g, e in zip(got, expect)), [(g, e) for g, e in zip(got, expect) if not fnmatch.fnmatchcase(g, e)]


# ---------------------------------------------------------------------------------------------- the public C++ surface
def test_eigen_overloads_compile_against_the_reference_headers(tmp_path):
    """with Eigen / OpenCV headers on the include path (the stand-ins of oracle/ref_shim here) the reference's
    decomposeProjectionMatrix(MatrixXd, Matrix3d&, Matrix3d&, Vector3d&) is available; both helpers run on the host"""
    so = build.build()
    src = tmp_path / "h.cpp"
    src.write_text(r"""
#include "line3d.h"
#include <cstdio>
int main() {
    Eigen::MatrixXd P(3, 4);
    const double v[12] = {1200, 3, 640, 10, 0, 1100, 480, -20, 0, 0, 1, 2};
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 4; ++c) P(r, c) = v[4 * r + c];
    Eigen::Matrix3d K, R; Eigen::Vector3d t;
    L3DPP::Line3D::decomposeProjectionMatrix(P, K, R, t);
    const L3DPP::Matrix3d Q = L3DPP::Line3D::rotationFromRPY(0.1, 0.2, 0.3);
    for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) std::printf("%.17g %.17g ", K(r, c), R(r, c));
    std::printf("%.17g %.17g %.17g %.17g\n", t(0), t(1), t(2), Q(1, 2));
    return 0;
}
""")
    exe = tmp_path / "h"
    cmd = ["g++", "-std=c++17", "-Wall", "-Werror", str(src), "-I" + os.path.join(ROOT, "include"), "-I" + os.path.join(ROOT, "oracle", "ref_shim"),
           "-L" + os.path.dirname(so), "-ll3d_b200", "-Wl,-rpath," + os.path.dirname(so), "-o", str(exe)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = [float(x) for x in r.stdout.split()]
    P = np.array([[1200, 3, 640, 10], [0, 1100, 480, -20], [0, 0, 1, 2.0]])
    K, R, t = line3d.decompose_projection_matrix(P)
    assert np.array_equal(np.array(out[0:18:2]), K.ravel()) and np.array_equal(np.array(out[1:18:2]), R.ravel()) and np.array_equal(np.array(out[18:21]), t)
    assert out[21] == line3d.rotation_from_rpy(0.1, 0.2, 0.3)[1, 2]


def test_sfm_frontend_example_compiles_and_reads_every_format(scene, tmp_path):
    """examples/sfm_frontend.cpp (the mavmap / OpenMVG / Pix4D frontends on include/line3d.h + include/line3d_io.h) compiles
    warning-free against the public headers; without a GPU it stops with "no usable CUDA device" instead of computing on the CPU"""
    so = build.build()
    exe = tmp_path / "sfm_frontend"
    cmd = ["g++", "-std=c++17", "-Wall", "-Wextra", "-Werror", os.path.join(ROOT, "examples", "sfm_frontend.cpp"), "-I" + os.path.join(ROOT, "include"),
           "-L" + os.path.dirname(so), "-ll3d_b200", "-Wl,-rpath," + os.path.dirname(so), "-o", str(exe)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    scene.write_mavmap(tmp_path / "m.txt")
    (tmp_path / "o.json").write_text(scene.openmvg_text())
    segs = tmp_path / "segs"
    segs.mkdir()
    r = subprocess.run([str(exe), "nothing", str(tmp_path / "m.txt"), str(segs), str(tmp_path)], capture_output=True, text=True)
    assert r.returncode == 2 and "usage" in r.stderr
    for fmt, model in (("mavmap", tmp_path / "m.txt"), ("openmvg", tmp_path / "o.json")):
        r = subprocess.run([str(exe), fmt, str(model), str(segs), str(tmp_path)], capture_output=True, text=True)
        if _has_gpu():
            assert r.returncode == 1 and "fewer than three usable images" in r.stderr, (fmt, r.returncode, r.stderr)
        else:
            assert r.returncode == 3 and "no usable CUDA device" in r.stderr, (fmt, r.returncode, r.stderr)
    (tmp_path / "bad.json").write_text("{")
    r = subprocess.run([str(exe), "openmvg", str(tmp_path / "bad.json"), str(segs), str(tmp_path)], capture_output=True, text=True)
    assert r.returncode == 1 and "bad.json" in r.stderr
