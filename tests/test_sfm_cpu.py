"""The mavmap, OpenMVG and Pix4D readers and the two frontend helpers without a GPU (include/line3d_io.h, csrc/line3d_sfm.cc,
DESIGN.md §6b): a synthetic scene written in each format is read back exactly, malformed input is rejected with a message, and the
reader file alone survives every malformed file under AddressSanitizer."""
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

from line3dpp_b200 import build, capi, line3d
from tests import sfm_scene as ss

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
// argv: M <file> (mavmap), O <file> (OpenMVG), P <folder> (Pix4D, prefix "proj"); prints one line per input
int main(int argc, char** argv)
{
    for (int i = 1; i + 1 < argc; i += 2) {
        std::string err;
        std::vector<L3DPP::SfMCamera> v;
        bool ok;
        if (argv[i][0] == 'M') ok = L3DPP::readMavmap(argv[i + 1], v, &err);
        else if (argv[i][0] == 'O') ok = L3DPP::readOpenMVG(argv[i + 1], v, &err);
        else ok = L3DPP::readPix4D(argv[i + 1], "proj", v, &err);
        std::printf("%s %zu %d\n", ok ? "ok" : "err", v.size(), (int)err.empty());
    }
    return 0;
}
"""


def test_readers_under_address_sanitizer(scene, tmp_path):
    """csrc/line3d_sfm.cc alone, built with ASan + UBSan, on a valid and every malformed input; allocations above 64 MB count as
    errors.  The Pix4D projects stop at the (stand-in) device step or earlier."""
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
    env = dict(os.environ, ASAN_OPTIONS="max_allocation_size_mb=64:allocator_may_return_null=0:detect_leaks=1")
    r = subprocess.run([str(exe)] + args, capture_output=True, text=True, env=env)
    assert r.returncode == 0 and "Sanitizer" not in r.stderr, r.stderr[-2000:]
    assert r.stdout.split("\n")[:-1] == expect


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
