"""The reference's binary files without a GPU (include/line3d_io.h, csrc/line3d_bin.cc, DESIGN.md §6a): the .bin result file of
save3DLinesAsBIN against the reference's own file, the segment cache layout, the cache file name, and malformed input."""
import hashlib
import lzma
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

from line3dpp_b200 import capi, line3d
from tests import nvm_util as nu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE_SHA = "7035690410a16185ea055e1b49bbaf9a6b8444fc96297830667b500c25024b67"   # the reference's <name>.bin, uncompressed


@pytest.fixture(scope="module")
def ref_bin():
    data = lzma.decompress(open(os.path.join(nu.G, "ref_lines_v1.bin.xz"), "rb").read())
    assert hashlib.sha256(data).hexdigest() == FIXTURE_SHA
    return data


@pytest.fixture()
def ref_path(ref_bin, tmp_path):
    p = tmp_path / "ref.bin"
    p.write_bytes(ref_bin)
    return p


def test_reference_bin_reads_and_matches_the_txt_result(ref_path):
    d = line3d.read_lines_bin(ref_path)
    assert (len(d["lines"]), len(d["segments"]), len(d["residuals"])) == (2489, 2501, 17603)
    segs3d, seg_line, res = nu.load_fixture()
    # the .txt result of the same run (one text line per 3D line, in order): same segments within its 6 significant digits
    mine = np.concatenate([d["segments"]["p1"], d["segments"]["p2"]], 1)
    assert mine.shape == segs3d.shape
    assert np.all(np.abs(mine - segs3d) <= 5e-6 * np.abs(mine) + 1e-12), np.abs(mine - segs3d).max()
    assert np.array_equal(d["segments"]["line"], seg_line)
    assert np.array_equal(np.stack([d["residuals"]["line"], d["residuals"]["cam"], d["residuals"]["seg"]], 1), res[:, :3].astype(np.int64))
    assert np.array_equal(d["lines"]["nseg"], np.bincount(seg_line, minlength=len(d["lines"])))
    # Segment3D fields as the reference computed them: valid, dir = unit(P2 - P1), length = |P2 - P1| in float
    for s in (d["segments"], d["clusters"]):
        assert s["valid"].all()
        v = s["p2"] - s["p1"]
        n = np.linalg.norm(v, axis=1)
        np.testing.assert_allclose(s["dir"], v / n[:, None], rtol=0, atol=1e-12)
        np.testing.assert_allclose(s["length"], n.astype(np.float32), rtol=1e-6)
    # the reference view is one of the cluster's residual cameras
    starts = np.r_[0, np.cumsum(d["lines"]["nres"])[:-1]]
    for i in range(0, len(d["lines"]), 97):
        cams = d["residuals"]["cam"][starts[i]:starts[i] + d["lines"]["nres"][i]]
        assert d["lines"]["reference_view"][i] in cams


def test_reference_bin_is_rewritten_byte_for_byte(ref_path, tmp_path):
    d = line3d.read_lines_bin(ref_path)
    out = tmp_path / "out.bin"
    line3d.write_lines_bin(out, d)
    assert hashlib.sha256(out.read_bytes()).hexdigest() == FIXTURE_SHA
    e = line3d.read_lines_bin(out)
    for k in d:
        assert d[k].tobytes() == e[k].tobytes(), k


def test_empty_result_file_layout(tmp_path):
    p = tmp_path / "empty.bin"
    line3d.write_lines_bin(p, dict(lines=np.zeros(0, line3d.LINE_DT), clusters=np.zeros(0, line3d.BIN_SEG_DT),
                                   segments=np.zeros(0, line3d.BIN_SEG_DT), residuals=np.zeros(0, line3d.RESID_DT)))
    assert p.read_bytes() == HEADER + b"\0" + b"\0" * 4 + struct.pack("<QI", 0, 0)
    assert len(line3d.read_lines_bin(p)["lines"]) == 0


# ---------------------------------------------------------------------------------------------- segment cache
HEADER = struct.pack("<Q", 22) + b"serialization::archive" + struct.pack("<H", 10) + bytes([4, 8, 4, 8]) + struct.pack("<i", 1)


def expected_cache(segs):
    """DataArray<float4>(n, 1) as Boost writes it (dataArray.h:104-125, 355-374): class info, width, height, real width (rows padded to
    32 bytes), CPU pitch and stride, GPU pitch and stride (0), then real_width float4s, each after the float4 class info once"""
    n = len(segs)
    real = n + (1 if (16 * n) % 32 else 0)
    b = HEADER + b"\0" + struct.pack("<I", 0) + struct.pack("<IIIQQQQ", n, 1, real, 16 * real, real, 0, 0)
    if real:
        b += b"\0" + struct.pack("<I", 0)
    pad = np.zeros((real - n, 4), np.float32)
    return b + np.concatenate([np.asarray(segs, np.float32).reshape(-1, 4), pad]).astype("<f4").tobytes()


@pytest.mark.parametrize("n", [0, 1, 2, 3, 3000])
def test_segment_cache_layout_and_round_trip(tmp_path, n):
    rng = np.random.default_rng(n)
    segs = rng.uniform(0, 3072, (n, 4)).astype(np.float32)
    p = tmp_path / "c.bin"
    line3d.write_segment_cache(p, segs)
    assert p.read_bytes() == expected_cache(segs)
    back = line3d.read_segment_cache(p)
    assert back.shape == (n, 4) and back.tobytes() == segs.tobytes()


def test_segment_cache_path_matches_cv2_resize():
    z = np.load(os.path.join(nu.G, "cv2_resize_shapes_v1.npz"))
    for (w, h, m), (rw, rh) in zip(z["sizes"], z["shapes"]):
        assert line3d.segment_cache_path("/data/run", 17, w, h, m) == f"/data/run/L3D++_data/segments_L3D++_17_{rw}x{rh}_3000.bin", (w, h, m)


# ---------------------------------------------------------------------------------------------- malformed input
def _patched(data, off, b):
    return data[:off] + b + data[off + len(b):]


def bad_result_files(data):
    """(name, bytes) variants of a valid result file that must all be rejected"""
    out = [(f"truncated_{n}", data[:n]) for n in (0, 7, 29, 31, 35, 39, 44, 52, 56, 83, 100, 1000, len(data) // 2, len(data) - 1)]
    out += [("signature_bitflip", _patched(data, 10, bytes([data[10] ^ 0x04]))),
            ("signature_length", _patched(data, 0, struct.pack("<Q", 23))),
            ("library_version_7", _patched(data, 30, struct.pack("<H", 7))),
            ("sizeof_long_4", _patched(data, 33, bytes([4]))),
            ("sizeof_double_4", _patched(data, 35, bytes([4]))),
            ("byte_order", _patched(data, 36, struct.pack(">i", 1))),
            ("tracking_on", _patched(data, 40, bytes([1]))),
            ("class_version", _patched(data, 41, struct.pack("<I", 3))),
            ("line_count_huge", _patched(data, 45, struct.pack("<Q", 1 << 62))),
            ("line_count_plus_one", _patched(data, 45, struct.pack("<Q", 2490))),
            ("item_version", _patched(data, 53, struct.pack("<I", 1))),
            ("segment_count_huge", _patched(data, 67, struct.pack("<Q", 0xFFFFFFFFFFFFFFFF))),
            ("segment_count_oversized", _patched(data, 67, struct.pack("<Q", len(data)))),
            ("bool_2", _patched(data, 88, bytes([2]))),
            ("trailing_byte", data + b"\0")]
    return out


def bad_cache_files(data):
    out = [(f"truncated_{n}", data[:n]) for n in (0, 39, 44, 52, 60, 80, 85, len(data) - 1)]
    out += [("signature_bitflip", _patched(data, 8, b"S")),
            ("sizeof_int_8", _patched(data, 32, bytes([8]))),
            ("height_2", _patched(data, 49, struct.pack("<I", 2))),
            ("real_width_huge", _patched(data, 53, struct.pack("<I", 0xFFFFFFFF))),
            ("width_over_real", _patched(data, 45, struct.pack("<I", 5))),
            ("stride_mismatch", _patched(data, 65, struct.pack("<Q", 7))),
            ("trailing_byte", data + b"\0")]
    return out


def test_malformed_result_files_are_rejected(ref_bin, tmp_path):
    for name, b in bad_result_files(ref_bin):
        p = tmp_path / f"{name}.bin"
        p.write_bytes(b)
        with pytest.raises(capi.L3DError) as e:
            line3d.read_lines_bin(p)
        assert str(p) in str(e.value), (name, str(e.value))
    with pytest.raises(capi.L3DError, match="cannot open"):
        line3d.read_lines_bin(tmp_path / "missing.bin")


def test_malformed_segment_caches_are_rejected(tmp_path):
    good = tmp_path / "good.bin"
    line3d.write_segment_cache(good, np.arange(12, dtype=np.float32).reshape(3, 4))
    for name, b in bad_cache_files(good.read_bytes()):
        p = tmp_path / f"{name}.bin"
        p.write_bytes(b)
        with pytest.raises(capi.L3DError) as e:
            line3d.read_segment_cache(p)
        assert str(p) in str(e.value), (name, str(e.value))


def test_writers_report_an_unwritable_folder(tmp_path):
    with pytest.raises(capi.L3DError, match="cannot open"):
        line3d.write_segment_cache(tmp_path / "no" / "such" / "dir.bin", np.zeros((2, 4), np.float32))
    with pytest.raises(capi.L3DError, match="cannot open"):
        line3d.write_lines_bin(tmp_path / "no" / "dir.bin", dict(lines=np.zeros(0, line3d.LINE_DT), clusters=np.zeros(0, line3d.BIN_SEG_DT),
                                                                  segments=np.zeros(0, line3d.BIN_SEG_DT), residuals=np.zeros(0, line3d.RESID_DT)))


ASAN_DRIVER = r"""
#include "line3d_io.h"
#include <cstdio>
#include <cstring>
// argv: L <file> (result file) or S <file> (segment cache) pairs; prints one line per file
int main(int argc, char** argv)
{
    for (int i = 1; i + 1 < argc; i += 2) {
        std::string err;
        bool ok; size_t n = 0;
        if (argv[i][0] == 'L') { std::vector<L3DPP::FinalLine3D> v; ok = L3DPP::read3DLinesBIN(argv[i + 1], v, &err); n = v.size(); }
        else { std::vector<L3DPP::Vec4f> v; ok = L3DPP::readSegmentCache(argv[i + 1], v, &err); n = v.size(); }
        std::printf("%s %zu %d\n", ok ? "ok" : "err", n, (int)err.empty());
    }
    return 0;
}
"""


def test_readers_under_address_sanitizer(ref_bin, tmp_path):
    """the readers alone (csrc/line3d_bin.cc needs no CUDA), built with ASan + UBSan, on the valid and every malformed file; allocations
    above 64 MB count as errors, so a count that is believed before it is checked fails here too"""
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no g++")
    drv = tmp_path / "drv.cc"
    drv.write_text(ASAN_DRIVER)
    exe = tmp_path / "drv"
    cmd = [gxx, "-std=c++17", "-g", "-O1", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "line3dpp_b200", "csrc", "line3d_bin.cc"), str(drv), "-o", str(exe)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        if "sanitize" in r.stderr or "asan" in r.stderr:
            pytest.skip("this compiler cannot build with AddressSanitizer: " + r.stderr[-300:])
        raise AssertionError(r.stderr)
    good_cache = tmp_path / "cache.bin"
    line3d.write_segment_cache(good_cache, np.arange(12, dtype=np.float32).reshape(3, 4))
    args, expect = [], []
    (tmp_path / "ref.bin").write_bytes(ref_bin)
    args += ["L", str(tmp_path / "ref.bin"), "S", str(good_cache)]
    expect += ["ok 2489 1", "ok 3 1"]
    for kind, variants in (("L", bad_result_files(ref_bin)), ("S", bad_cache_files(good_cache.read_bytes()))):
        for name, b in variants:
            p = tmp_path / f"{kind}_{name}.bin"
            p.write_bytes(b)
            args += [kind, str(p)]
            expect.append("err 0 0")
    env = dict(os.environ, ASAN_OPTIONS="max_allocation_size_mb=64:allocator_may_return_null=0:detect_leaks=1")
    r = subprocess.run([str(exe)] + args, capture_output=True, text=True, env=env)
    assert r.returncode == 0 and "Sanitizer" not in r.stderr, r.stderr[-2000:]
    assert r.stdout.split("\n")[:-1] == expect
