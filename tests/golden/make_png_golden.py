"""Generate tests/golden/ref_png_v1.npz: what OpenCV 4.13's cv2.imread(path, IMREAD_GRAYSCALE) returns for every PNG fixture of
tests/test_png_cpu.py / tests/test_png_gpu.py.  Needs cv2 and Pillow; run from the repository root:

    python tests/golden/make_png_golden.py

Cases:
  writer_*    tests/png_model.py's writer (png_model.writer_cases): only the parameters and the SHA-256 of the file are stored, the
              bytes are rebuilt by the tests
  cv2_* pil_* cv2.imencode (compression levels 0 / 1 / 9) and Pillow files: grey, RGB, RGBA, palette, 16-bit; bytes stored, since zlib's
              output differs between zlib versions
For each: cv2's output size and the SHA-256 of its bytes, and the bytes themselves when the output has at most 4096 pixels.
Before anything is written, the model (png_model.decode_gray) must reproduce cv2 on every case, and libpng's gamma path as the model
states it must reproduce cv2 on all 2^24 RGB triples for every gamma value of the fixtures.  Also stored: the files the parser
rejects, with their reasons (png_model.reject_files), after checking that the model rejects each with that reason.
"""
import hashlib
import io
import json
import os
import struct
import sys
import zlib

import cv2
import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests import png_model as pm  # noqa: E402


def imdecode(b):
    return cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_GRAYSCALE)


def test_image(w, h, seed):
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    img = np.stack([(x * 255 // max(w - 1, 1)), (y * 255 // max(h - 1, 1)), ((x + y) * 3) % 256], axis=2).astype(np.int64)
    img += rng.integers(-20, 21, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


def encoder_cases():
    out = []
    bgr = test_image(97, 61, 1)
    for lv in (0, 1, 9):
        out.append((f"cv2_rgb_level{lv}", cv2.imencode(".png", bgr, [cv2.IMWRITE_PNG_COMPRESSION, lv])[1].tobytes()))
        out.append((f"cv2_grey_level{lv}", cv2.imencode(".png", bgr[:, :, 1], [cv2.IMWRITE_PNG_COMPRESSION, lv])[1].tobytes()))
    bgra = np.concatenate([bgr, test_image(97, 61, 2)[:, :, :1]], 2)
    out.append(("cv2_rgba", cv2.imencode(".png", bgra)[1].tobytes()))
    out.append(("cv2_rgb16", cv2.imencode(".png", bgr.astype(np.uint16) * 257 + 3)[1].tobytes()))
    out.append(("cv2_grey16", cv2.imencode(".png", bgr[:, :, 0].astype(np.uint16) * 201)[1].tobytes()))
    rgb = bgr[:, :, ::-1]
    for name, im, kw in [("pil_rgb", Image.fromarray(rgb), {}), ("pil_grey", Image.fromarray(rgb[:, :, 0]), {"compress_level": 9}),
                         ("pil_palette", Image.fromarray(rgb).quantize(200), {}), ("pil_palette_4bit", Image.fromarray(rgb).quantize(16), {"bits": 4}),
                         ("pil_rgba", Image.fromarray(np.concatenate([rgb, rgb[:, :, :1]], 2)), {}),
                         ("pil_grey_alpha", Image.fromarray(np.stack([rgb[:, :, 0], rgb[:, :, 1]], 2)), {}),
                         ("pil_1bit", Image.fromarray(rgb[:, :, 0] > 128), {}), ("pil_rgb_adam7_opt", Image.fromarray(rgb), {"optimize": True})]:
        f = io.BytesIO()
        im.save(f, "PNG", **kw)
        out.append((name, f.getvalue()))
    return out


def check_gamma_all_triples(gammas):
    v = np.arange(1 << 24, dtype=np.int64)
    rgb = np.stack([v >> 16, (v >> 8) & 255, v & 255], -1).reshape(4096, 4096, 3)
    for g in gammas:
        pre = [(b"sRGB", b"\0")] if g == "srgb" else [(b"gAMA", struct.pack(">I", g))]
        b = pm.write_png(rgb, 2, 8, pre=pre, compress=lambda r: zlib.compress(r, 1))
        want = imdecode(b)
        got = pm.decode_gray(b)
        bad = int((want != got).sum())
        print(f"gamma {g}: {bad} of 2^24 triples differ")
        assert bad == 0


def pack(blobs):
    """byte strings -> (one uint8 array, offsets [n + 1]); no pickled objects in the archive"""
    off = np.cumsum([0] + [len(b) for b in blobs]).astype(np.int64)
    return np.frombuffer(b"".join(blobs), np.uint8).copy(), off


def main():
    cases = []
    for name, p in pm.writer_cases():
        cases.append(("writer_" + name, "writer", json.dumps(p, sort_keys=True), pm.build_case(p)))
    for name, b in encoder_cases():
        cases.append((name, "bytes", "", b))
    names, kinds, params, blobs, fsha, widths, heights, osha, small = [], [], [], [], [], [], [], [], []
    for name, kind, p, b in cases:
        want = imdecode(b)
        assert want is not None, name
        got = pm.decode_gray(b)
        assert got.shape == want.shape and np.array_equal(got, want), (name, got.shape, want.shape)
        names.append(name); kinds.append(kind); params.append(p)
        blobs.append(b if kind == "bytes" else b"")
        fsha.append(hashlib.sha256(b).hexdigest())
        heights.append(want.shape[0]); widths.append(want.shape[1])
        osha.append(hashlib.sha256(np.ascontiguousarray(want).tobytes()).hexdigest())
        small.append(want.tobytes() if want.size <= 4096 else b"")
    gammas = sorted({int(c[1], 16) for _, k, p, _ in cases if k == "writer" for c in json.loads(p).get("pre", []) if c[0] == "gAMA"})
    check_gamma_all_triples(gammas + ["srgb"])
    rej = pm.reject_files()
    for name, b, why in rej:
        try:
            pm.parse(b)
            raise AssertionError(name + " parses")
        except pm.PngError as e:
            assert str(e) == why, (name, str(e), why)
    print(len(cases), "cases,", len(rej), "rejections")
    blob, off = pack(blobs)
    oblob, ooff = pack(small)
    rblob, roff = pack([r[1] for r in rej])
    np.savez_compressed(os.path.join(HERE, "ref_png_v1.npz"), name=np.array(names), kind=np.array(kinds), params=np.array(params),
                        files=blob, file_off=off, sha_file=np.array(fsha), width=np.array(widths), height=np.array(heights),
                        sha_out=np.array(osha), out=oblob, out_off=ooff, reject_name=np.array([r[0] for r in rej]), reject_file=rblob,
                        reject_off=roff, reject_reason=np.array([r[2] for r in rej]))


if __name__ == "__main__":
    main()
