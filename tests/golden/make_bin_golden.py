"""Builds the fixtures of the binary-file tests (tests/test_bin_cpu.py) from the reference's test data and cv2:

    python tests/golden/make_bin_golden.py

ref_lines_v1.bin.xz: testdata/Line3D++_ref/<name>.bin of the non-optimized run (the reference's save3DLinesAsBIN, a Boost
  binary_oarchive of std::vector<FinalLine3D>), lzma-compressed.
cv2_resize_shapes_v1.npz: the image size cv::resize(img, out, Size(), s, s) gives with s = float(max_img_width) / float(max(w, h)),
  the <w>x<h> of the reference's segment cache file names (line3D.cc:271-300), for a handful of sizes.

It also round-trips the OPTIMIZED run's .bin through the library's reader and writer and checks byte equality and its counts;
that file is not committed.
"""
import hashlib
import lzma
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
REF = "/root/reference/testdata/Line3D++_ref"
NAME = "Line3D++__W_FULL__N_10__sigmaP_2.5__sigmaA_10__epiOverlap_0.25__kNN_10__{}vis_3.bin"
OUT = os.path.dirname(os.path.abspath(__file__))

# (width, height, max_img_width): landscape and portrait, exact halves (cvRound rounds them to even), no-resize cases
SIZES = [(3072, 2304, 1920), (2304, 3072, 1920), (3072, 2304, 3072), (3072, 2304, 4000), (3072, 2304, -1), (2000, 1333, 1000),
         (1333, 2000, 1000), (4000, 2998, 1000), (4000, 2994, 1000), (5472, 3648, 1234), (801, 800, 800), (4912, 3264, 2047),
         (6000, 4000, 999), (1920, 1080, 1280)]


def resize_shape(w, h, max_w):
    import cv2
    if max_w <= 0 or max(w, h) <= max_w:
        return w, h
    s = float(np.float32(max_w) / np.float32(max(w, h)))
    out = cv2.resize(np.zeros((h, w), np.uint8), None, fx=s, fy=s)
    return out.shape[1], out.shape[0]


def main():
    from line3dpp_b200 import line3d
    plain = open(os.path.join(REF, NAME.format("")), "rb").read()
    with open(os.path.join(OUT, "ref_lines_v1.bin.xz"), "wb") as f:
        f.write(lzma.compress(plain, preset=9 | lzma.PRESET_EXTREME))
    print("ref_lines_v1.bin.xz:", len(plain), "bytes, sha256", hashlib.sha256(plain).hexdigest())
    opt = os.path.join(REF, NAME.format("OPTIMIZED__"))
    d = line3d.read_lines_bin(opt)
    assert (len(d["lines"]), len(d["segments"]), len(d["residuals"])) == (2490, 2503, 17606)
    tmp = os.path.join(OUT, "_optimized_roundtrip.bin")
    try:
        line3d.write_lines_bin(tmp, d)
        assert open(tmp, "rb").read() == open(opt, "rb").read(), "OPTIMIZED .bin does not round-trip byte for byte"
    finally:
        if os.path.exists(tmp):
            os.remove(tmp)
    print("OPTIMIZED .bin: 2490 lines, 2503 segments, 17606 residuals, byte-identical after read + write")
    sizes = np.array(SIZES, np.int32)
    shapes = np.array([resize_shape(*s) for s in SIZES], np.int32)
    np.savez_compressed(os.path.join(OUT, "cv2_resize_shapes_v1.npz"), sizes=sizes, shapes=shapes)
    for s, o in zip(SIZES, shapes):
        print(s, "->", tuple(o))


if __name__ == "__main__":
    sys.exit(main())
