"""Writes tests/golden/ref_image_prep_v1.npz: the grey, resized image OpenCV makes for the reference's detectLineSegments
(line3D.cc:249-289: cvtColor(CV_RGB2GRAY), then cv::resize(gray, out, Size(), s, s) with INTER_LINEAR when max_img_width asks for it)
on the cases below, and checks the numpy restatement (tests/image_prep_model.py) against cv2 first: over all 2^24 RGB triples and on
every case.

Needs cv2 (any CPU machine).  The inputs come from tests/image_prep_model.make_image (seeded), so only digests, the small outputs and a
sample of the grey table are stored.  Per case:
  <name>/params        width, height, channels, max_img_width, seed, row padding (bytes the GPU tests add to every source row)
  <name>/out_size      (width, height) of cv2's output
  <name>/cv_sha        SHA-256 of cv2's output
  <name>/cv_out        cv2's output itself for outputs of at most 64k pixels
and gray_rgb (uint8 [n, 3]) / gray_val (uint8 [n]): a random sample of cvtColor's table, cv2_version / cv2_cpu.

    python tests/golden/make_image_prep_golden.py
"""
import os
import re
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests import image_prep_model as pm  # noqa: E402

OUT = os.path.join(HERE, "ref_image_prep_v1.npz")

# name: (width, height, channels, max_img_width, row padding); what each reaches is in the comment
CASES = {
    "gray_noresize": (1000, 800, 1, -1, 0),          # max_img_width <= 0: grey copy
    "rgb_fits": (1200, 900, 3, 1200, 5),              # max(w, h) == max_img_width: grey conversion only
    "rgb_landscape": (1037, 811, 3, 1000, 0),         # INTER_LINEAR, landscape
    "gray_portrait": (813, 1290, 1, 777, 3),          # INTER_LINEAR, portrait, padded rows
    "rgb_half": (1000, 803, 3, 500, 0),               # step exactly 2: INTER_AREA 2x2, last row from one source row
    "gray_half_portrait": (999, 1002, 1, 501, 7),     # step exactly 2, portrait, last column from one source column
    "rgb_half_even": (1600, 1200, 3, 800, 0),         # step exactly 2, no border
    "gray_third": (1200, 900, 1, 400, 0),             # integer step 3 stays INTER_LINEAR
    "rgb_quarter": (1600, 1200, 3, 400, 9),           # integer step 4 stays INTER_LINEAR
    "gray_w50": (97, 61, 1, 50, 0),                   # output width 50 (not a multiple of 8 or 16)
    "rgb_w129": (333, 517, 3, 200, 1),                # output width 129 (odd), portrait
    "gray_lastrow_256": (401, 300, 1, 256, 0),        # last output row: second tap clamped with its weight kept
    "rgb_lastrow_200": (401, 300, 3, 200, 2),
    "rgb_vsfm_1920": (3072, 2304, 3, 1920, 0),        # a VisualSfM-size image with max_img_width 1920
    "gray_vsfm_1920": (3072, 2304, 1, 1920, 11),
}
SMALL = 1 << 16


def cpu_features(cv2):
    info = cv2.getBuildInformation()
    lines = [m.group(0).strip() for m in re.finditer(r"^\s*(Baseline|Dispatched code generation):.*$", info, re.M)]
    return " | ".join(lines)


def cv_prepare(cv2, img, mw):
    """line3D.cc:251-289 in cv2"""
    g = cv2.cvtColor(img, cv2.COLOR_RGB2GRAY) if img.ndim == 3 else img.copy()
    h, w = g.shape
    if mw > 0 and max(w, h) > mw:
        s = np.float32(mw) / np.float32(max(w, h))
        g = cv2.resize(g, None, fx=float(s), fy=float(s))       # default INTER_LINEAR
    return g


def main():
    import cv2
    v = np.arange(1 << 24, dtype=np.uint32)
    rgb = np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    table = cv2.cvtColor(rgb, cv2.COLOR_RGB2GRAY)
    assert np.array_equal(pm.gray(rgb), table), "the grey model differs from cv2 somewhere in the 2^24 triples"
    pick = np.random.default_rng(7).choice(1 << 24, 4096, replace=False)
    out = {"cv2_version": np.array(cv2.__version__), "cv2_cpu": np.array(cpu_features(cv2)), "cases": np.array(list(CASES)),
           "gray_rgb": rgb.reshape(-1, 3)[pick], "gray_val": table.reshape(-1)[pick]}
    for i, (name, (w, h, c, mw, pad)) in enumerate(CASES.items()):
        img = pm.make_image(h, w, c, seed=100 + i)
        ref = cv_prepare(cv2, img, mw)
        model = pm.prepare(img, mw)
        assert ref.shape == model.shape and np.array_equal(ref, model), name
        assert (ref.shape[1], ref.shape[0]) == pm.prepared_size(w, h, mw)[:2], name
        P = f"{name}/"
        out[P + "params"] = np.array([w, h, c, mw, 100 + i, pad], np.int64)
        out[P + "out_size"] = np.array([ref.shape[1], ref.shape[0]], np.int64)
        out[P + "cv_sha"] = np.array(pm.sha(ref))
        if ref.size <= SMALL:
            out[P + "cv_out"] = ref
        print(f"{name:20s} {w}x{h}x{c} max_img_width {mw:5d} -> {ref.shape[1]}x{ref.shape[0]}: model == cv2")
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes;", out["cv2_version"], out["cv2_cpu"])


if __name__ == "__main__":
    main()
