"""JPEG decoding without a GPU (DESIGN.md §4c): the integer restatement (tests/jpeg_model.py) against what OpenCV 4.13's imread returned
(tests/golden/ref_jpeg_v1.npz, from tests/golden/make_jpeg_golden.py), the header-only size functions on every fixture, every rejected
kind of file with its message, and the library's refusal to decode without a GPU."""
import ctypes
import hashlib
import json
import os
import re
import struct

import numpy as np
import pytest

from tests import jpeg_model as jm

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(os.path.join(GOLD, "ref_jpeg_v1.npz")))


def case_bytes(g, i):
    """the file of case i: rebuilt by the writer, stored, or a photo next to the golden file"""
    kind = str(g["kinds"][i])
    if kind == "writer":
        return jm.build_case(json.loads(str(g["params"][i])))
    if kind == "photo":
        return open(os.path.join(GOLD, str(g["params"][i])), "rb").read()
    return g[f"file_{i}"].tobytes()


def _cases():
    g = dict(np.load(os.path.join(GOLD, "ref_jpeg_v1.npz")))
    return [(i, str(n)) for i, n in enumerate(g["names"])]


CASES = _cases()


@pytest.mark.parametrize("i,name", [c for c in CASES if not c[1].startswith("photo")], ids=[c[1] for c in CASES if not c[1].startswith("photo")])
def test_model_reproduces_opencv(gold, i, name):
    data = case_bytes(gold, i)
    assert hashlib.sha256(data).hexdigest() == str(gold["sha_file"][i]), "the writer no longer builds the same file"
    out = jm.decode_gray(data)
    assert out.shape == (int(gold["height"][i]), int(gold["width"][i]))
    assert hashlib.sha256(out.tobytes()).hexdigest() == str(gold["sha_out"][i])
    if f"out_{i}" in gold:
        np.testing.assert_array_equal(out, gold[f"out_{i}"])


def test_fixtures_reach_what_they_are_for(gold):
    """the writer cases cover the paths the golden file claims: saturated IDCT outputs, DC-only blocks whose 16-bit shift wraps, 16-bit
    Huffman codes, DC differences of size 11, ZRL runs, stuffed bytes before restart markers, every orientation"""
    names = [str(n) for n in gold["names"]]
    wc = jm.writer_cases()
    ext = jm.build_case(wc["extreme_q255"])
    info = jm.parse(ext)
    co = jm.decode_y_coefs(ext, info).astype(np.int64).reshape(-1, 8, 8)
    deq = jm._i16(co * info["comps"][0]["q"].reshape(8, 8))
    dc_only = ~np.any(co[:, 1:, :], axis=(1, 2))
    assert np.any(dc_only & (np.abs(deq[:, 0, 0]) >= 8192)), "no DC-only block wraps in the 16-bit shift"
    px = jm.idct_islow(co.reshape(-1, 64), info["comps"][0]["q"])
    assert np.any(px == 0) and np.any(px == 255)
    h16 = jm.parse(jm.build_case(wc["huff16"]))
    assert any(t["ac"][0][15] > 0 or t["dc"][0][15] > 0 for t in h16["scans"][0]["comps"]), "no 16-bit Huffman code"
    dc11 = jm.parse(jm.build_case(wc["dc_size11"]))
    assert 11 in dc11["scans"][0]["comps"][0]["dc"][1]
    zrl = jm.parse(jm.build_case(wc["zrl_sparse"]))
    assert 0xF0 in zrl["scans"][0]["comps"][0]["ac"][1]
    for o in range(1, 9):
        assert f"writer_exif_{o}_ii" in names and f"writer_exif_{o}_mm" in names


@pytest.mark.parametrize("i,name", CASES, ids=[c[1] for c in CASES])
def test_sizes_after_orientation(gold, tmp_path, i, name):
    from line3dpp_b200 import capi, line3d
    data = case_bytes(gold, i)
    want = (int(gold["width"][i]), int(gold["height"][i]))
    assert capi.jpeg_info(data) == want
    p = tmp_path / "f.jpg"
    p.write_bytes(data)
    assert line3d.jpeg_size(p) == want


def _sof(data):
    """offset of the SOF marker's payload (precision byte)"""
    i = 2
    while True:
        m, ln = data[i + 1], struct.unpack(">H", data[i + 2:i + 4])[0]
        if m in (0xC0, 0xC1, 0xC2, 0xC3, 0xC5, 0xC9):
            return i + 4
        i += 2 + ln


def _patch(data, off, vals):
    b = bytearray(data)
    b[off:off + len(vals)] = bytes(vals)
    return bytes(b)


def _base(**kw):
    p = dict(w=40, h=24, sampling="420", seed=7)
    p.update(kw)
    return jm.build_case(p)


def _first(data, marker):
    i = 2
    while data[i + 1] != marker:
        i += 2 + struct.unpack(">H", data[i + 2:i + 4])[0]
    return i


def _rejects():
    base = _base()
    s = _sof(base)
    sos = _first(base, 0xDA)
    out = {
        "not_jpeg": (b"\x89PNG\r\n\x1a\n" + base[8:], "not a JPEG file (no SOI marker)"),
        "progressive_sof2": (_base(sof=0xC2), "progressive JPEG is not supported"),
        "lossless_sof3": (_base(sof=0xC3), "lossless JPEG is not supported"),
        "hierarchical_sof5": (_base(sof=0xC5), "hierarchical JPEG is not supported"),
        "arithmetic_sof9": (_base(sof=0xC9), "arithmetic coding is not supported"),
        "arithmetic_dac": (base[:2] + b"\xFF\xCC\x00\x04\x00\x10" + base[2:], "arithmetic coding is not supported"),
        "precision_12": (_patch(base, s, [12]), "12-bit precision is not supported"),
        "dnl_height_0": (_patch(base, s + 1, [0, 0]), "DNL markers are not supported"),
        "dnl_marker": (base[:-2] + b"\xFF\xDC\x00\x04\x00\x18\xFF\xD9", "DNL markers are not supported"),
        "components_2": (_patch(base, s + 5, [2]), "2 components are not supported"),
        "components_4": (_patch(base, s + 5, [4]), "4 components are not supported"),
        "rgb_adobe_0": (_base(jfif=False, adobe=0), "RGB JPEG is not supported"),
        "rgb_ids": (_base(jfif=False, ids=[82, 71, 66]), "RGB JPEG is not supported"),
        "y_below_max_sampling": (jm.write_jpeg(24, 16, [(1, 1, 0), (2, 2, 1), (1, 1, 1)],
                                               jm.random_coefs(np.random.default_rng(1), 24, 16, [(1, 1, 0), (2, 2, 1), (1, 1, 1)]),
                                               {0: jm.std_q(), 1: jm.std_q()}), "Y is not at the largest sampling factors"),
        "side_40000": (_patch(base, s + 3, [40000 >> 8, 40000 & 255]), "image side outside [1, 32767]"),
        "missing_huffman": (_patch(base, sos + 6, [0x33]), "missing Huffman table"),
        "missing_quant": (_patch(base, s + 8, [3]), "missing quantisation table"),
        "truncated_scan": (base[:sos + 30], "truncated entropy-coded data"),
        "truncated_header": (base[:s + 3], "truncated marker segment"),
        "missing_eoi": (base[:-2] + b"\xFF\xFE\x00\x03x", "missing EOI marker"),
        "no_frame": (base[:2] + b"\xFF\xD9", "no frame header"),
        "component_without_scan": (_base(scans=[[0], [1]]), "a component has no scan"),
        "bad_restart_number": (None, "corrupt restart markers"),
        "restart_count": (None, "corrupt restart markers"),
        "garbage_between_markers": (base[:2] + b"\x00" + base[2:], "corrupt data between markers"),
    }
    r = bytearray(_base(restart=2))
    k = bytes(r).index(b"\xFF\xD1")
    r[k + 1] = 0xD5
    out["bad_restart_number"] = (bytes(r), out["bad_restart_number"][1])
    r = _base(restart=2)
    k = r.index(b"\xFF\xD1")
    out["restart_count"] = (r[:k] + r[k + 2:], out["restart_count"][1])
    return out


REJECTS = _rejects()


@pytest.mark.parametrize("name", sorted(REJECTS))
def test_rejected_with_its_reason(tmp_path, name):
    from line3dpp_b200 import capi, line3d
    data, msg = REJECTS[name]
    with pytest.raises(jm.JpegError, match=re.escape(msg)):
        jm.parse(data)
    w, h = ctypes.c_int32(), ctypes.c_int32()
    assert capi.lib().l3d_jpeg_info(data, len(data), ctypes.byref(w), ctypes.byref(h)) == -1
    p = tmp_path / "f.jpg"
    p.write_bytes(data)
    with pytest.raises(capi.L3DError) as e:
        line3d.jpeg_size(p)
    assert str(e.value) == f"{p}: {msg}" or (str(e.value).startswith(f"{p}: {msg}")), str(e.value)


@pytest.mark.parametrize("name", ["cv2_progressive", "pil_progressive"])
def test_encoder_progressive_files_are_rejected(gold, tmp_path, name):
    from line3dpp_b200 import capi, line3d
    p = tmp_path / "f.jpg"
    p.write_bytes(gold[f"reject_{name}"].tobytes())
    with pytest.raises(capi.L3DError, match="progressive JPEG is not supported"):
        line3d.jpeg_size(p)


def test_unreadable_file(tmp_path):
    from line3dpp_b200 import capi, line3d
    with pytest.raises(capi.L3DError, match="cannot open file"):
        line3d.jpeg_size(tmp_path / "missing.jpg")


def test_jpeg_desc_layout(tmp_path):
    """capi.JpegDesc has l3d_jpeg_desc's layout"""
    import subprocess
    from line3dpp_b200 import capi
    inc = os.path.join(os.path.dirname(GOLD), "..", "include")
    fields = [f for f, _ in capi.JpegDesc._fields_]
    src = tmp_path / "l.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "l3d_capi.h"\nint main(void)\n{\n    printf("%zu\\n", sizeof(l3d_jpeg_desc));\n'
                   + "".join(f'    printf("%zu %zu\\n", offsetof(l3d_jpeg_desc, {f}), sizeof(((l3d_jpeg_desc*)0)->{f}));\n' for f in fields)
                   + "    return 0;\n}\n")
    exe = tmp_path / "l"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", inc, str(src), "-o", str(exe)], check=True)
    got = [tuple(int(x) for x in line.split()) for line in subprocess.check_output([str(exe)], text=True).splitlines()]
    assert got[0] == (ctypes.sizeof(capi.JpegDesc),)
    assert got[1:] == [(getattr(capi.JpegDesc, f).offset, getattr(capi.JpegDesc, f).size) for f in fields]


def _has_gpu():
    import torch
    return torch.cuda.is_available()


def test_decoding_needs_a_gpu(gold, tmp_path):
    from line3dpp_b200 import capi, line3d
    if _has_gpu():
        pytest.skip("a GPU is present (tests/test_jpeg_gpu.py decodes)")
    with pytest.raises(capi.L3DError, match="no usable CUDA device"):
        capi.Context(0)
    p = tmp_path / "f.jpg"
    p.write_bytes(case_bytes(gold, 0))
    with pytest.raises(capi.L3DError, match="no usable CUDA device"):
        line3d.read_jpeg_gray(p)
