"""PNG decoding without a GPU (DESIGN.md §4d): tests/png_model.py against what OpenCV 4.13's imread(IMREAD_GRAYSCALE) returned for every
fixture of tests/golden/ref_png_v1.npz, the chunk parser behind l3d_png_info / readPNGSize on every fixture and every rejection reason,
and readImageSize's choice between the JPEG and the PNG reader."""
import hashlib
import json
import os

import numpy as np
import pytest

from tests import png_model as pm

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
_G = np.load(os.path.join(GOLDEN, "ref_png_v1.npz"))
CASES = [(i, str(n)) for i, n in enumerate(_G["name"])]
REJECTS = [(i, str(n)) for i, n in enumerate(_G["reject_name"])]


@pytest.fixture(scope="module")
def gold():
    return _G


def _blob(g, key, i):
    off = g[key + "_off"]
    data = g[{"file": "files", "reject": "reject_file"}.get(key, key)]
    return data[off[i]:off[i + 1]].tobytes()


def case_bytes(g, i):
    """the file of case i: stored bytes, or rebuilt by the writer from its parameters (checked against the stored digest)"""
    b = _blob(g, "file", i) if str(g["kind"][i]) == "bytes" else pm.build_case(json.loads(str(g["params"][i])))
    assert hashlib.sha256(b).hexdigest() == str(g["sha_file"][i]), str(g["name"][i])
    return b


def reject_bytes(g, i):
    return _blob(g, "reject", i)


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.mark.parametrize("i,name", CASES, ids=[c[1] for c in CASES])
def test_model_equals_opencv(gold, i, name):
    out = pm.decode_gray(case_bytes(gold, i))
    assert out.shape == (int(gold["height"][i]), int(gold["width"][i]))
    assert sha(out) == str(gold["sha_out"][i])
    small = _blob(gold, "out", i)
    if small:
        assert out.tobytes() == small


def test_fixtures_cover_the_format(gold):
    params = [json.loads(str(p)) for p, k in zip(gold["params"], gold["kind"]) if str(k) == "writer"]
    got = {(p["ct"], p["depth"], p.get("interlace", 0)) for p in params}
    for ct, depths in pm.LEGAL.items():
        for d in depths:
            assert (ct, d, 0) in got and (ct, d, 1) in got
    deflates = {p.get("deflate") for p in params}
    assert {"stored", "fixed", "dyn_chain", "single_dist", "no_dist", "far", "overlap", "block_in_row"} <= deflates
    assert {(o, be) for o in range(1, 9) for be in ("ii", "mm")} <= {(int(str(n).split("_")[2]), str(n).split("_")[3])
                                                                      for n in gold["name"] if str(n).startswith("writer_exif_") and str(n)[12].isdigit()
                                                                      and len(str(n).split("_")) == 4}


def test_writer_layouts_are_what_they_claim():
    """the special DEFLATE layouts hold what their names say, read back by zlib"""
    raw = bytes(np.random.default_rng(3).integers(0, 15, 1600, dtype=np.uint8))
    for kind in ("stored", "fixed", "dyn_chain", "single_dist", "no_dist", "overlap", "block_in_row"):
        assert pm.zlib.decompress(pm.special_deflate(kind, raw)) == raw, kind
    big = bytes(np.random.default_rng(4).integers(0, 256, 70000, dtype=np.uint8))
    z = pm.special_deflate("stored", big)
    assert pm.zlib.decompress(z) == big
    assert z[2:7] == b"\x00\x00\x00\xff\xff"          # the empty stored block first
    toks = pm.lz77(raw, window=31)
    assert all(t[1] <= 31 for t in toks if isinstance(t, tuple)) and any(t[0] > t[1] for t in toks if isinstance(t, tuple))


@pytest.fixture(scope="module")
def lib():
    from line3dpp_b200 import capi
    return capi


@pytest.mark.parametrize("i,name", CASES, ids=[c[1] for c in CASES])
def test_png_info(lib, gold, i, name):
    assert lib.png_info(case_bytes(gold, i)) == (int(gold["width"][i]), int(gold["height"][i]))


@pytest.mark.parametrize("i,name", REJECTS, ids=[c[1] for c in REJECTS])
def test_rejection_reason(lib, gold, tmp_path, i, name):
    from line3dpp_b200 import line3d
    b = reject_bytes(gold, i)
    with pytest.raises(lib.L3DError):
        lib.png_info(b)
    p = tmp_path / (name + ".png")
    p.write_bytes(b)
    with pytest.raises(lib.L3DError) as e:
        line3d.png_size(p)
    assert str(e.value) == f"{p}: {gold['reject_reason'][i]}"
    with pytest.raises(pm.PngError, match="^" + __import__("re").escape(str(gold["reject_reason"][i])) + "$"):
        pm.parse(b)


def test_png_size_and_image_size_dispatch(gold, tmp_path):
    from line3dpp_b200 import capi, line3d
    k = [i for i, n in CASES if n == "writer_exif_6_ii"][0]
    p = tmp_path / "a.png"
    p.write_bytes(case_bytes(gold, k))
    assert line3d.png_size(p) == line3d.image_size(p) == (int(gold["width"][k]), int(gold["height"][k]))
    jpg = os.path.join(GOLDEN, "jpeg_photo_0.jpg")
    assert line3d.image_size(jpg) == line3d.jpeg_size(jpg) == (3072, 2304)
    with pytest.raises(capi.L3DError, match="not a PNG file"):
        line3d.png_size(jpg)
    t = tmp_path / "notes.txt"
    t.write_bytes(b"hello, world")
    with pytest.raises(capi.L3DError, match="not a JPEG or PNG file"):
        line3d.image_size(t)
    with pytest.raises(capi.L3DError, match="cannot open file"):
        line3d.image_size(tmp_path / "missing.png")
