"""JPEG decoding on the GPU (l3d_decode_jpeg_gray_u8, DESIGN.md §4c) against what OpenCV 4.13's imread(IMREAD_GRAYSCALE) returned for
every fixture of tests/golden/ref_jpeg_v1.npz: through host and device outputs, one file at a time and all in one batch, with untouched
row padding, calls rejected before any write, the batched file reader, and the device chain decode -> undistort -> prepare."""
import ctypes as C
import hashlib
import json

import numpy as np
import pytest

from tests import jpeg_model as jm
from tests.test_jpeg_cpu import CASES, REJECTS, case_bytes, gold  # noqa: F401  (gold: the fixture)

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture(scope="module")
def files(gold):  # noqa: F811
    return [case_bytes(gold, i) for i, _ in CASES]


@pytest.fixture(scope="module")
def ctx():
    from line3dpp_b200 import capi
    c = capi.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("i,name", CASES, ids=[c[1] for c in CASES])
def test_case_equals_opencv_host_and_device(ctx, gold, files, i, name):  # noqa: F811
    want = str(gold["sha_out"][i])
    host = ctx.decode_jpeg_gray([files[i]])[0]
    assert host.shape == (int(gold["height"][i]), int(gold["width"][i]))
    assert sha(host) == want
    dev = torch.empty(host.shape, dtype=torch.uint8, device="cuda")
    ctx.decode_jpeg_gray([files[i]], out=[dev])
    assert sha(dev.cpu().numpy()) == want


def test_one_batch_equals_one_by_one(ctx, gold, files):  # noqa: F811
    photos = [k for k, (_, n) in enumerate(CASES) if n.startswith("photo")]
    order = list(range(len(files))) + [photos[j % len(photos)] for j in range(64)]
    rng = np.random.default_rng(0)
    rng.shuffle(order)
    outs = ctx.decode_jpeg_gray([files[k] for k in order])
    for k, o in zip(order, outs):
        assert sha(o) == str(gold["sha_out"][k]), CASES[k][1]
    # the same batch into device outputs
    dev = [torch.empty(o.shape, dtype=torch.uint8, device="cuda") for o in outs]
    ctx.decode_jpeg_gray([files[k] for k in order], out=dev)
    for k, d in zip(order, dev):
        assert sha(d.cpu().numpy()) == str(gold["sha_out"][k]), CASES[k][1]


def test_row_padding_stays_untouched(ctx, gold, files):  # noqa: F811
    pick = [k for k, (_, n) in enumerate(CASES) if n in ("writer_420_17x9", "writer_exif_6_ii", "cv2_rst3", "writer_grey_1x1", "photo_0")]
    host, dev = [], []
    for k in pick:
        h, w = int(gold["height"][k]), int(gold["width"][k])
        host.append(np.full((h, w + 13), 0xA5, np.uint8)[:, :w])
        dev.append(torch.full((h, w + 40), 0x5A, dtype=torch.uint8, device="cuda")[:, :w])
    ctx.decode_jpeg_gray([files[k] for k in pick], out=host)
    ctx.decode_jpeg_gray([files[k] for k in pick], out=dev)
    for k, o, d in zip(pick, host, dev):
        assert sha(o) == str(gold["sha_out"][k])
        assert np.all(o.base[:, o.shape[1]:] == 0xA5)
        full = d.as_strided((d.shape[0], d.stride(0)), (d.stride(0), 1)).cpu().numpy()
        assert sha(full[:, :d.shape[1]]) == str(gold["sha_out"][k])
        assert np.all(full[:, d.shape[1]:] == 0x5A)


def _descs(files, outs, on_device):
    from line3dpp_b200 import capi
    descs = (capi.JpegDesc * len(files))()
    for i, (f, o) in enumerate(zip(files, outs)):
        w, h = capi.jpeg_info(f)
        descs[i].data = C.cast(C.c_char_p(f), C.c_void_p).value
        descs[i].size = len(f)
        descs[i].dst = o.data_ptr() if on_device else o.ctypes.data
        descs[i].dst_pitch = o.stride(0) if on_device else o.strides[0]
        descs[i].out_width, descs[i].out_height = w, h
    return descs


@pytest.mark.parametrize("on_device", [0, 1])
@pytest.mark.parametrize("bad", ["null_dst", "out_size", "pitch", "progressive", "no_data", "corrupt_entropy", "short_segment"])
def test_a_bad_descriptor_fails_the_call_and_writes_nothing(ctx, files, bad, on_device):
    """one bad entry (index 4) among good ones: the call fails naming it; nothing is written (device outputs excepted when the coded
    data is found corrupt on the GPU, after the kernels ran)"""
    from line3dpp_b200 import capi
    batch = [files[k] for k, (_, n) in enumerate(CASES) if n.startswith("writer_sampling") or n.startswith("cv2_q")]
    idx = 4
    good = jm.build_case(dict(w=40, h=24, sampling="420", restart=2, seed=7))
    if bad == "corrupt_entropy":       # a run of 1 bits at the start of the scan: the all-ones code is never assigned
        k = good.index(b"\xFF\xDA")
        k += 2 + (good[k + 2] << 8 | good[k + 3])
        batch[idx] = good[:k + 4] + b"\xFF\x00" * 8 + good[k + 20:]
    elif bad == "short_segment":       # the first restart interval loses its last bytes
        k = good.index(b"\xFF\xD0")
        batch[idx] = good[:k - 6] + good[k:]
    sizes = [capi.jpeg_info(f) for f in batch]
    if on_device:
        outs = [torch.full((h, w), 7, dtype=torch.uint8, device="cuda") for w, h in sizes]
    else:
        outs = [np.full((h, w), 7, np.uint8) for w, h in sizes]
    descs = _descs(batch, outs, on_device)
    progressive = REJECTS["progressive_sof2"][0]
    if bad == "null_dst":
        descs[idx].dst = None
    elif bad == "out_size":
        descs[idx].out_width += 1
    elif bad == "pitch":
        descs[idx].dst_pitch = descs[idx].out_width - 1
    elif bad == "progressive":
        descs[idx].data, descs[idx].size = C.cast(C.c_char_p(progressive), C.c_void_p).value, len(progressive)
    elif bad == "no_data":
        descs[idx].data = None
    with pytest.raises(capi.L3DError, match=f"image {idx}: "):
        ctx.decode_jpeg_gray_descs(descs, on_device)
    if bad in ("corrupt_entropy", "short_segment") and on_device:
        return
    for o in outs:
        assert np.all((o.cpu().numpy() if on_device else o) == 7)


def test_readers_decode_the_readable_files(gold, files, tmp_path):  # noqa: F811
    from line3dpp_b200 import capi, line3d
    names = ["cv2_q50", "writer_exif_7_mm", "photo_1"]
    paths = []
    for n in names:
        k = [c[1] for c in CASES].index(n)
        p = tmp_path / f"{n}.jpg"
        p.write_bytes(files[k])
        paths.append(p)
    paths.insert(1, tmp_path / "missing.jpg")
    bad = tmp_path / "progressive.jpg"
    bad.write_bytes(REJECTS["progressive_sof2"][0])
    paths.append(bad)
    errors = []
    outs = line3d.read_jpeg_gray(paths, errors=errors)
    assert outs[1] is None and "cannot open file" in errors[1]
    assert outs[4] is None and errors[4] == f"{bad}: progressive JPEG is not supported"
    for j, n in zip((0, 2, 3), names):
        k = [c[1] for c in CASES].index(n)
        assert errors[j] == "" and sha(outs[j]) == str(gold["sha_out"][k])
    with pytest.raises(capi.L3DError, match="cannot open file"):
        line3d.read_jpeg_gray(paths)
    assert sha(line3d.read_jpeg_gray(paths[0])) == sha(outs[0])


def test_device_chain_decode_undistort_prepare(ctx, gold, files):  # noqa: F811
    """decode -> l3d_undistort_u8 -> l3d_prepare_gray_u8, all on_device=1: the bytes of cv2's imread -> remap -> resize"""
    from line3dpp_b200 import capi
    chain = json.loads(str(gold["chain"]))
    k = [c[1] for c in CASES].index("photo_0")
    h, w = int(gold["height"][k]), int(gold["width"][k])
    img = torch.empty((h, w), dtype=torch.uint8, device="cuda")
    ctx.decode_jpeg_gray([files[k]], out=[img])
    D = chain["D"]
    und = torch.empty_like(img)
    ud = (capi.UndistortDesc * 1)()
    ud[0] = capi.make_undistort_desc(w, h, 1, chain["K"], radial=(D[0], D[1], D[4]), tangential=(D[2], D[3]), src=img.data_ptr(), src_pitch=w,
                                     dst=und.data_ptr(), dst_pitch=w)
    ctx.undistort_device(ud)
    ow, oh, _ = capi.image_prep_size(w, h, chain["max_img_width"])
    assert (oh, ow) == tuple(int(v) for v in gold["chain_prep_shape"])
    prep = torch.empty((oh, ow), dtype=torch.uint8, device="cuda")
    pd = (capi.ImagePrepDesc * 1)()
    pd[0] = capi.make_image_prep_desc(w, h, 1, chain["max_img_width"], und.data_ptr(), w, prep.data_ptr(), ow)
    ctx.prepare_gray_device(pd)
    ctx.sync()
    assert sha(und.cpu().numpy()) == str(gold["chain_undistort_sha"])
    assert sha(prep.cpu().numpy()) == str(gold["chain_prep_sha"])
