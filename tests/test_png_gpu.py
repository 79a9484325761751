"""PNG decoding on the GPU (l3d_decode_png_gray_u8, DESIGN.md §4d) against what OpenCV 4.13's imread(IMREAD_GRAYSCALE) returned for
every fixture of tests/golden/ref_png_v1.npz: through host and device outputs, alone and in one batch, mixed with JPEG files through
readImagesGray; untouched row padding; calls rejected before any write; every corrupt-stream kind found on the GPU and named; all
2^24 RGB triples against the grey formula; a photo-size round trip; and the device chain decode -> undistort -> prepare."""
import ctypes as C
import hashlib
import os
import zlib

import numpy as np
import pytest

from tests import png_model as pm
from tests.test_png_cpu import CASES, GOLDEN, case_bytes, gold, reject_bytes  # noqa: F401  (gold: the fixture)

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
    host = ctx.decode_png_gray([files[i]])[0]
    assert host.shape == (int(gold["height"][i]), int(gold["width"][i]))
    assert sha(host) == want
    dev = torch.empty(host.shape, dtype=torch.uint8, device="cuda")
    ctx.decode_png_gray([files[i]], out=[dev])
    assert sha(dev.cpu().numpy()) == want


def test_one_batch_equals_one_by_one(ctx, gold, files):  # noqa: F811
    order = list(range(len(files))) * 2
    np.random.default_rng(0).shuffle(order)
    outs = ctx.decode_png_gray([files[k] for k in order])
    for k, o in zip(order, outs):
        assert sha(o) == str(gold["sha_out"][k]), CASES[k][1]
    dev = [torch.empty(o.shape, dtype=torch.uint8, device="cuda") for o in outs]
    ctx.decode_png_gray([files[k] for k in order], out=dev)
    for k, d in zip(order, dev):
        assert sha(d.cpu().numpy()) == str(gold["sha_out"][k]), CASES[k][1]


def test_mixed_jpeg_and_png_through_read_image_gray(gold, files, tmp_path):  # noqa: F811
    from line3dpp_b200 import line3d
    from tests.test_jpeg_cpu import CASES as JCASES, case_bytes as jcase
    jg = np.load(os.path.join(GOLDEN, "ref_jpeg_v1.npz"))
    paths, want = [], []
    for j, (k, n) in enumerate(CASES):
        p = tmp_path / f"p{j}.png"
        p.write_bytes(files[k])
        paths.append(p)
        want.append(str(gold["sha_out"][k]))
    for j, (k, n) in enumerate(JCASES):
        p = tmp_path / f"j{j}.jpg"
        p.write_bytes(jcase(jg, k))
        paths.insert(2 * j, p)
        want.insert(2 * j, str(jg["sha_out"][k]))
    other = tmp_path / "notes.txt"
    other.write_bytes(b"neither")
    bad = tmp_path / "bad.png"
    bad.write_bytes(reject_bytes(gold, [str(n) for n in gold["reject_name"]].index("iccp")))
    errors = []
    outs = line3d.read_image_gray(paths + [other, bad], errors=errors)
    for o, e, w, p in zip(outs, errors, want, paths):
        assert e == "" and sha(o) == w, p
    assert outs[-2] is None and errors[-2] == f"{other}: not a JPEG or PNG file"
    assert outs[-1] is None and errors[-1] == f"{bad}: iCCP colour profiles are not supported"
    assert sha(line3d.read_png_gray(paths[1])) == want[1]
    assert sha(line3d.read_image_gray(paths[0])) == want[0]


def test_row_padding_stays_untouched(ctx, gold, files):  # noqa: F811
    pick = [k for k, n in CASES if n in ("writer_exif_6_ii", "writer_ct2_d16_adam7", "writer_adam7_grey_1x1", "pil_palette", "writer_deflate_stored")]
    host, dev = [], []
    for k in pick:
        h, w = int(gold["height"][k]), int(gold["width"][k])
        host.append(np.full((h, w + 13), 0xA5, np.uint8)[:, :w])
        dev.append(torch.full((h, w + 40), 0x5A, dtype=torch.uint8, device="cuda")[:, :w])
    ctx.decode_png_gray([files[k] for k in pick], out=host)
    ctx.decode_png_gray([files[k] for k in pick], out=dev)
    for k, o, d in zip(pick, host, dev):
        assert sha(o) == str(gold["sha_out"][k])
        assert np.all(o.base[:, o.shape[1]:] == 0xA5)
        full = d.as_strided((d.shape[0], d.stride(0)), (d.stride(0), 1)).cpu().numpy()
        assert sha(full[:, :d.shape[1]]) == str(gold["sha_out"][k])
        assert np.all(full[:, d.shape[1]:] == 0x5A)


def _descs(files, outs, on_device):
    from line3dpp_b200 import capi
    descs = (capi.PngDesc * len(files))()
    for i, (f, o) in enumerate(zip(files, outs)):
        w, h = capi.png_info(f)
        descs[i].data = C.cast(C.c_char_p(f), C.c_void_p).value
        descs[i].size = len(f)
        descs[i].dst = o.data_ptr() if on_device else o.ctypes.data
        descs[i].dst_pitch = o.stride(0) if on_device else o.strides[0]
        descs[i].out_width, descs[i].out_height = w, h
    return descs


@pytest.mark.parametrize("on_device", [0, 1])
@pytest.mark.parametrize("bad", ["null_dst", "out_size", "pitch", "rejected_file", "no_data"])
def test_a_bad_descriptor_fails_the_call_and_writes_nothing(ctx, gold, files, bad, on_device):  # noqa: F811
    from line3dpp_b200 import capi
    batch = [files[k] for k, n in CASES if n.startswith("writer_ct")][:8]
    idx = 4
    sizes = [capi.png_info(f) for f in batch]
    if on_device:
        outs = [torch.full((h, w), 7, dtype=torch.uint8, device="cuda") for w, h in sizes]
    else:
        outs = [np.full((h, w), 7, np.uint8) for w, h in sizes]
    descs = _descs(batch, outs, on_device)
    rejected = reject_bytes(gold, [str(n) for n in gold["reject_name"]].index("chrm"))
    if bad == "null_dst":
        descs[idx].dst = None
    elif bad == "out_size":
        descs[idx].out_width += 1
    elif bad == "pitch":
        descs[idx].dst_pitch = descs[idx].out_width - 1
    elif bad == "rejected_file":
        descs[idx].data, descs[idx].size = C.cast(C.c_char_p(rejected), C.c_void_p).value, len(rejected)
    elif bad == "no_data":
        descs[idx].data = None
    with pytest.raises(capi.L3DError, match=f"image {idx}: "):
        ctx.decode_png_gray_descs(descs, on_device)
    for o in outs:
        assert np.all((o.cpu().numpy() if on_device else o) == 7)


CORRUPT = pm.corrupt_streams()


@pytest.mark.parametrize("name,data,reason", CORRUPT, ids=[c[0] for c in CORRUPT])
def test_corrupt_stream_is_found_on_the_gpu_and_named(ctx, files, name, data, reason):
    """the corrupt file at index 2 of a good batch: the call fails naming it and its reason; host outputs stay untouched"""
    from line3dpp_b200 import capi
    pm.parse(data)                                       # the headers are fine: only the GPU can find the fault
    with pytest.raises(pm.PngError):
        pm.decode_gray(data)
    batch = files[:2] + [data] + files[2:4]
    outs = [np.full((h, w), 7, np.uint8) for w, h in (capi.png_info(f) for f in batch)]
    with pytest.raises(capi.L3DError, match="image 2: " + reason.replace("(", r"\(").replace(")", r"\)")):
        ctx.decode_png_gray(batch, out=outs)
    for o in outs:
        assert np.all(o == 7)
    ctx.decode_png_gray(files[:2], out=outs[:2])        # the context is still usable


def test_all_rgb_triples(ctx):
    v = np.arange(1 << 24, dtype=np.int64)
    rgb = np.stack([v >> 16, (v >> 8) & 255, v & 255], -1).reshape(4096, 4096, 3)
    b = pm.write_png(rgb, 2, 8, filters=(0, 1, 2, 3, 4), compress=lambda r: zlib.compress(r, 1))
    out = ctx.decode_png_gray([b])[0]
    assert np.array_equal(out, pm.rgb_to_gray8(rgb[..., 0], rgb[..., 1], rgb[..., 2]))


def test_photo_round_trip(ctx):
    """a 3072 x 2304 photo decoded from JPEG on the GPU, written as a grey PNG by the writer, decodes to the same bytes"""
    with open(os.path.join(GOLDEN, "jpeg_photo_0.jpg"), "rb") as f:
        grey = ctx.decode_jpeg_gray([f.read()])[0]
    for filters, il in (((0, 1, 2, 3, 4), 0), ((4,), 1)):
        b = pm.write_png(grey, 0, 8, interlace=il, filters=filters)
        assert np.array_equal(ctx.decode_png_gray([b])[0], grey)


def test_device_chain_equals_host_chain(ctx, gold, files):  # noqa: F811
    """PNG decode -> l3d_undistort_u8 -> l3d_prepare_gray_u8 with on_device=1 gives the bytes of the same calls in host mode"""
    from line3dpp_b200 import capi
    with open(os.path.join(GOLDEN, "jpeg_photo_1.jpg"), "rb") as f:
        grey = ctx.decode_jpeg_gray([f.read()])[0]
    png = pm.write_png(grey, 0, 8, filters=(1, 4), pre=[(b"eXIf", pm.exif_block(6))])
    w, h = capi.png_info(png)
    K = [[2400.0, 0, w / 2 - 0.5], [0, 2410.0, h / 2 + 0.25], [0, 0, 1]]
    radial, tang, mw = (-0.12, 0.05, 0.0), (0.001, -0.0007), 1920
    ow, oh, _ = capi.image_prep_size(w, h, mw)
    # host mode, one call at a time
    img = ctx.decode_png_gray([png])[0]
    und_h = np.empty_like(img)
    ud = (capi.UndistortDesc * 1)()
    ud[0] = capi.make_undistort_desc(w, h, 1, K, radial=radial, tangential=tang, src=img.ctypes.data, src_pitch=w, dst=und_h.ctypes.data, dst_pitch=w)
    ctx.L.l3d_undistort_u8(ctx.h, 1, ud, 0)
    prep_h = np.empty((oh, ow), np.uint8)
    pd = (capi.ImagePrepDesc * 1)()
    pd[0] = capi.make_image_prep_desc(w, h, 1, mw, und_h.ctypes.data, w, prep_h.ctypes.data, ow)
    ctx.L.l3d_prepare_gray_u8(ctx.h, 1, pd, 0)
    # device mode
    dimg = torch.empty((h, w), dtype=torch.uint8, device="cuda")
    ctx.decode_png_gray([png], out=[dimg])
    und = torch.empty_like(dimg)
    ud[0] = capi.make_undistort_desc(w, h, 1, K, radial=radial, tangential=tang, src=dimg.data_ptr(), src_pitch=w, dst=und.data_ptr(), dst_pitch=w)
    ctx.undistort_device(ud)
    prep = torch.empty((oh, ow), dtype=torch.uint8, device="cuda")
    pd[0] = capi.make_image_prep_desc(w, h, 1, mw, und.data_ptr(), w, prep.data_ptr(), ow)
    ctx.prepare_gray_device(pd)
    ctx.sync()
    assert np.array_equal(dimg.cpu().numpy(), img) and np.array_equal(img, np.ascontiguousarray(grey.T[:, ::-1]))
    assert np.array_equal(und.cpu().numpy(), und_h)
    assert np.array_equal(prep.cpu().numpy(), prep_h)
