"""Generate tests/golden/ref_jpeg_v1.npz: what OpenCV 4.13's cv2.imread(path, IMREAD_GRAYSCALE) returns for every JPEG fixture of
tests/test_jpeg_cpu.py / tests/test_jpeg_gpu.py.  Needs cv2 and Pillow; run from the repository root:

    python tests/golden/make_jpeg_golden.py [TESTDATA_DIR]

TESTDATA_DIR: Line3D++'s testdata folder; its img000055.jpg and img000056.jpg are copied here as jpeg_photo_0.jpg / _1.jpg.  Without
it the committed copies are used.

Cases:
  writer_*    tests/jpeg_model.py's writer (jpeg_model.writer_cases): only the parameters and the SHA-256 of the file are stored, the
              bytes are rebuilt from the seed
  cv2_*       cv2.imencode files (qualities, sampling factors, restart intervals, optimised tables, grey input); bytes stored
  pil_*       Pillow-encoded files; bytes stored
  photo_*     two of the reference's testdata photos (3072 x 2304, 4:2:0, no DRI), stored next to this file as jpeg_photo_*.jpg
For each: cv2's output size and the SHA-256 of its bytes, and the bytes themselves when the output has at most 4096 pixels.
Before anything is written, the model (jpeg_model.decode_gray) must reproduce cv2 on every case.
Also stored: encoder-made files that must be rejected (progressive), and the digest of cv2's imread -> remap (radtan lens) ->
INTER_LINEAR resize on the first photo, the path of the device-chaining test.
"""
import hashlib
import io
import json
import os
import sys
import tempfile

import cv2
import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from tests import jpeg_model as jm  # noqa: E402

PHOTOS = ["img000055.jpg", "img000056.jpg"]
# the device-chaining case: a radtan lens and the prep width (tests/test_jpeg_gpu.py)
CHAIN = dict(K=[[2400.0, 0, 1530.5], [0, 2410.0, 1160.25], [0, 0, 1]], D=[-0.12, 0.05, 0.001, -0.0007, 0.0], max_img_width=1920)


def imread_gray(b):
    fd, p = tempfile.mkstemp(suffix=".jpg")
    try:
        os.write(fd, b)
        os.close(fd)
        return cv2.imread(p, cv2.IMREAD_GRAYSCALE)
    finally:
        os.unlink(p)


def test_image(w, h, seed):
    """a smooth scene with edges and noise, BGR uint8"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    img = np.stack([(x * 255 // max(w - 1, 1)), (y * 255 // max(h - 1, 1)), ((x + y) * 3) % 256], axis=2).astype(np.int64)
    img[(x - w // 2) ** 2 + (y - h // 3) ** 2 < (min(w, h) // 4) ** 2] = [30, 200, 90]
    img += rng.integers(-20, 21, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


def encoder_cases():
    out = {}
    img = test_image(97, 61, 1)
    for q in (5, 25, 50, 75, 90, 100):
        out[f"cv2_q{q}"] = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q])[1].tobytes()
    for name in ("411", "420", "422", "440", "444"):
        sf = getattr(cv2, f"IMWRITE_JPEG_SAMPLING_FACTOR_{name}")
        out[f"cv2_sf{name}"] = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 85, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, sf])[1].tobytes()
    for ri in (1, 3, 7):
        out[f"cv2_rst{ri}"] = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_RST_INTERVAL, ri])[1].tobytes()
    out["cv2_optimize"] = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_OPTIMIZE, 1, cv2.IMWRITE_JPEG_QUALITY, 60])[1].tobytes()
    out["cv2_optimize_rst2_411"] = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_OPTIMIZE, 1, cv2.IMWRITE_JPEG_RST_INTERVAL, 2,
                                                              cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411])[1].tobytes()
    out["cv2_grey"] = cv2.imencode(".jpg", cv2.cvtColor(img, cv2.COLOR_BGR2GRAY), [cv2.IMWRITE_JPEG_QUALITY, 80])[1].tobytes()
    big = test_image(517, 389, 2)
    out["cv2_517x389"] = cv2.imencode(".jpg", big, [cv2.IMWRITE_JPEG_QUALITY, 92])[1].tobytes()
    pil = Image.fromarray(img[:, :, ::-1])
    for q, sub, opt in ((10, 2, False), (70, 1, False), (95, 0, True), (50, 2, True)):
        b = io.BytesIO()
        pil.save(b, "JPEG", quality=q, subsampling=sub, optimize=opt)
        out[f"pil_q{q}_sub{sub}_{'opt' if opt else 'std'}"] = b.getvalue()
    b = io.BytesIO()
    pil.convert("L").save(b, "JPEG", quality=65)
    out["pil_grey"] = b.getvalue()
    b = io.BytesIO()
    exif = Image.Exif()
    exif[0x0112] = 6
    pil.save(b, "JPEG", quality=80, exif=exif.tobytes())
    out["pil_exif6"] = b.getvalue()
    return out


def rejected_cases():
    img = test_image(64, 40, 3)
    b = io.BytesIO()
    Image.fromarray(img).save(b, "JPEG", progressive=True)
    return {"cv2_progressive": cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes(), "pil_progressive": b.getvalue()}


def main():
    names, kinds, params, sha_file, widths, heights, sha_out = [], [], [], [], [], [], []
    arrays = {}

    def add(name, kind, data, par=""):
        ref = imread_gray(data)
        assert ref is not None, name
        model = jm.decode_gray(data)
        assert model.shape == ref.shape and np.array_equal(model, ref), f"{name}: the model differs from cv2 in {(model != ref).sum()} pixels"
        i = len(names)
        names.append(name); kinds.append(kind); params.append(par)
        sha_file.append(hashlib.sha256(data).hexdigest())
        widths.append(ref.shape[1]); heights.append(ref.shape[0])
        sha_out.append(hashlib.sha256(np.ascontiguousarray(ref).tobytes()).hexdigest())
        if kind == "bytes":
            arrays[f"file_{i}"] = np.frombuffer(data, np.uint8)
        if ref.size <= 4096:
            arrays[f"out_{i}"] = ref
        print(f"{name}: {ref.shape[1]}x{ref.shape[0]}, {len(data)} bytes")

    stuffed = False
    for name, p in jm.writer_cases().items():
        data = jm.build_case(p)
        stuffed |= any(data[k] == 0xFF and data[k + 1] == 0 and data[k + 2] == 0xFF and 0xD0 <= data[k + 3] <= 0xD7 for k in range(len(data) - 3))
        add("writer_" + name, "writer", data, json.dumps(p))
    assert stuffed, "no fixture has a stuffed 0xFF right before a restart marker"
    for name, data in encoder_cases().items():
        add(name, "bytes", data)
    photos = []
    for k, f in enumerate(PHOTOS):
        dst = os.path.join(HERE, f"jpeg_photo_{k}.jpg")
        if len(sys.argv) > 1:
            with open(dst, "wb") as fo:
                fo.write(open(os.path.join(sys.argv[1], f), "rb").read())
        photos.append(open(dst, "rb").read())
        add(f"photo_{k}", "photo", photos[-1], os.path.basename(dst))
    rej = rejected_cases()
    for name, data in rej.items():
        arrays[f"reject_{name}"] = np.frombuffer(data, np.uint8)
    # the chaining case: imread -> initUndistortRectifyMap (fixed point) + remap -> resize as l3d_prepare_gray_u8 does it
    ref = imread_gray(photos[0])
    K, D = np.array(CHAIN["K"]), np.array(CHAIN["D"])
    m1, m2 = cv2.initUndistortRectifyMap(K, D, None, K, (ref.shape[1], ref.shape[0]), cv2.CV_16SC2)
    und = cv2.remap(ref, m1, m2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    s = np.float32(CHAIN["max_img_width"]) / np.float32(max(ref.shape))
    prep = cv2.resize(und, None, fx=float(s), fy=float(s), interpolation=cv2.INTER_LINEAR)
    np.savez_compressed(os.path.join(HERE, "ref_jpeg_v1.npz"), names=np.array(names), kinds=np.array(kinds), params=np.array(params),
                        sha_file=np.array(sha_file), width=np.array(widths), height=np.array(heights), sha_out=np.array(sha_out),
                        reject_names=np.array(sorted(rej)), chain=np.array(json.dumps(CHAIN)),
                        chain_undistort_sha=np.array(hashlib.sha256(und.tobytes()).hexdigest()),
                        chain_prep_sha=np.array(hashlib.sha256(np.ascontiguousarray(prep).tobytes()).hexdigest()),
                        chain_prep_shape=np.array(prep.shape), **arrays)
    print(f"{len(names)} cases")


if __name__ == "__main__":
    main()
