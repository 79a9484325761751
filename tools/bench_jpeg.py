"""Time JPEG decoding (l3d_decode_jpeg_gray_u8, DESIGN.md §4c) on the reference's 3072 x 2304 photos (tests/golden/jpeg_photo_*.jpg).

    python tools/bench_jpeg.py [--reps 5] [--batches 1,8,32,128] [--out FILE]

Per batch size (copies of the two photos), per image:
  - device time of each phase (k_jpeg_entropy, k_jpeg_idct) from torch.profiler's CUDA kernel records, and the wall time of the whole
    call with device outputs (parse, upload, both kernels, status check);
  - the end-to-end time of readJPEGsGray (files read, parsed, uploaded, decoded, downloaded; a context is created per call);
  - cv2.imdecode(..., IMREAD_GRAYSCALE) on one host thread and on nproc threads (Pillow's draft('L') decode when cv2 is absent: the same
    bytes).
Also the compressed bytes and pixels per image, the GPU's name and power limit, and the host's CPU count.  Prints one JSON object.
"""
import argparse
import io
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from line3dpp_b200 import capi, line3d  # noqa: E402

PHOTOS = [os.path.join(ROOT, "tests", "golden", f"jpeg_photo_{k}.jpg") for k in (0, 1)]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def host_decoder():
    try:
        import cv2
        return "cv2.imdecode", lambda b: cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_GRAYSCALE)
    except ImportError:
        from PIL import Image

        def pil(b):
            im = Image.open(io.BytesIO(b))
            im.draft("L", im.size)
            return np.asarray(im.convert("L"))
        return "PIL draft('L')", pil


def kernel_ms(prof, name):
    tot = 0.0
    for e in prof.key_averages():
        if e.key.startswith(name):
            tot += getattr(e, "device_time_total", 0.0) or getattr(e, "cuda_time_total", 0.0)
    return tot / 1000.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batches", default="1,8,32,128")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_jpeg: no CUDA device (nothing is measured without one)")
    files = [open(p, "rb").read() for p in PHOTOS]
    w, h = capi.jpeg_info(files[0])
    ctx = capi.Context(0)
    res = dict(gpu=gpu_info(), cpu_count=os.cpu_count(), width=w, height=h, pixels=w * h,
               compressed_bytes=[len(f) for f in files], reps=a.reps, batches={})
    ref = ctx.decode_jpeg_gray(files)
    for b in [int(x) for x in a.batches.split(",")]:
        batch = [files[j % 2] for j in range(b)]
        outs = [torch.empty((h, w), dtype=torch.uint8, device="cuda") for _ in range(b)]
        ctx.decode_jpeg_gray(batch, out=outs)                      # warm-up: buffers grown, modules loaded
        for j in (0, b - 1):
            assert np.array_equal(outs[j].cpu().numpy(), ref[j % 2])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(a.reps):
            ctx.decode_jpeg_gray(batch, out=outs)
        wall = (time.perf_counter() - t0) / a.reps
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(a.reps):
                ctx.decode_jpeg_gray(batch, out=outs)
            torch.cuda.synchronize()
        ent, idct = kernel_ms(prof, "k_jpeg_entropy") / a.reps, kernel_ms(prof, "k_jpeg_idct") / a.reps
        res["batches"][b] = dict(call_ms=wall * 1e3, call_ms_per_image=wall * 1e3 / b, entropy_ms=ent, idct_ms=idct,
                                 entropy_ms_per_image=ent / b, idct_ms_per_image=idct / b,
                                 idct_gpix_per_s=b * w * h / (idct * 1e-3) / 1e9 if idct > 0 else None)
        del outs
        print(json.dumps({"batch": b, **res["batches"][b]}), file=sys.stderr)
    # readJPEGsGray end to end, from files on disk
    tmp = tempfile.mkdtemp()
    try:
        paths = []
        for j in range(32):
            p = os.path.join(tmp, f"p{j}.jpg")
            shutil.copyfile(PHOTOS[j % 2], p)
            paths.append(p)
        e2e = {}
        for b in (1, 32):
            line3d.read_jpeg_gray(paths[:b])
            t0 = time.perf_counter()
            for _ in range(a.reps):
                line3d.read_jpeg_gray(paths[:b])
            e2e[b] = (time.perf_counter() - t0) / a.reps * 1e3 / b
        res["readJPEGsGray_ms_per_image"] = e2e
    finally:
        shutil.rmtree(tmp)
    name, dec = host_decoder()
    assert np.array_equal(dec(files[0]), ref[0]), "the host decoder's bytes differ"
    n1 = 8
    t0 = time.perf_counter()
    for j in range(n1):
        dec(files[j % 2])
    one = (time.perf_counter() - t0) / n1 * 1e3
    nproc = os.cpu_count() or 1
    batch = [files[j % 2] for j in range(4 * nproc)]
    with ThreadPoolExecutor(nproc) as ex:
        list(ex.map(dec, batch[:nproc]))
        t0 = time.perf_counter()
        list(ex.map(dec, batch))
        par = (time.perf_counter() - t0) / len(batch) * 1e3
    res["host"] = dict(decoder=name, ms_per_image_1_thread=one, ms_per_image_nproc_threads=par, threads=nproc)
    ctx.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
