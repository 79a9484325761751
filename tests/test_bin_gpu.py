"""save3DLinesAsBIN and addImage from the segment cache on the GPU (include/line3d.h, csrc/line3d_bin.cc): the .bin file of a real
reconstruction reads back bit for bit, and a run whose segments come from cache files equals the run that passed them explicitly."""
import os

import numpy as np
import pytest

from line3dpp_b200 import capi, line3d
from tests import nvm_util as nu
from tests import util

pytestmark = pytest.mark.gpu


def _add(L, inp, i, segs):
    w, h = inp["wh"][i]
    L.add_image(i, int(w), int(h), inp["K"][i], inp["R"][i], inp["t"][i], inp["median_depth"][i], inp["wps"][i], segs)


def _digest(L):
    s, r = L.segments3d(), L.residuals()
    return util.sha(s["line"], util.bits(s["p1"]), util.bits(s["p2"])), util.sha(r["line"], r["cam"], r["seg"])


@pytest.fixture(scope="module")
def inp():
    return nu.load_inputs()


@pytest.fixture(scope="module")
def explicit_run(inp):
    """the nvm inputs with their segments passed to addImage"""
    L = line3d.Line3D(neighbors_by_worldpoints=True, use_gpu=True)
    for i in range(inp["V"]):
        _add(L, inp, i, inp["segs"][i])
    L.match_images()
    L.reconstruct_3d_lines(3, False)
    yield L
    L.close()


def test_save_bin_reads_back_bit_for_bit(explicit_run, tmp_path):
    L = explicit_run
    L.save_bin(tmp_path)
    name = L.output_filename() + ".bin"
    assert name == "Line3D++__W_FULL__N_10__sigmaP_2.5__sigmaA_10__epiOverlap_0.25__kNN_10__vis_3.bin"
    assert os.listdir(tmp_path) == [name]
    got, mine = line3d.read_lines_bin(tmp_path / name), L.lines()
    assert len(mine["lines"]) == L.stats()["lines3D"] > 1000
    for k in ("lines", "clusters", "segments", "residuals"):
        assert got[k].tobytes() == mine[k].tobytes(), k
    s = L.segments3d()                                   # and the .bin agrees with the existing result accessors
    assert np.array_equal(util.bits(got["segments"]["p1"]), util.bits(s["p1"])) and np.array_equal(got["segments"]["line"], s["line"])
    assert np.array_equal(got["residuals"].tobytes(), L.residuals().tobytes())
    # writing what was read gives the same file again
    line3d.write_lines_bin(tmp_path / "again.bin", got)
    assert (tmp_path / "again.bin").read_bytes() == (tmp_path / name).read_bytes()


def test_save_bin_without_lines_writes_nothing(inp, tmp_path):
    L = line3d.Line3D(neighbors_by_worldpoints=True, use_gpu=True)
    _add(L, inp, 0, inp["segs"][0])
    with pytest.raises(capi.L3DError, match="no 3D lines"):
        L.save_bin(tmp_path)
    assert os.listdir(tmp_path) == []
    L.close()


def test_save_bin_reports_an_unwritable_folder(explicit_run, tmp_path):
    with pytest.raises(capi.L3DError, match="cannot open"):
        explicit_run.save_bin(tmp_path / "does" / "not" / "exist")


def test_add_image_reads_the_segment_cache(inp, explicit_run, tmp_path):
    """every view's segments written as the reference's cache files; addImage without segments then reconstructs exactly what the
    explicit-segment run reconstructs"""
    os.makedirs(tmp_path / "L3D++_data")
    for i in range(inp["V"]):
        w, h = inp["wh"][i]
        line3d.write_segment_cache(line3d.segment_cache_path(tmp_path, i, w, h, -1), inp["segs"][i])
    L = line3d.Line3D(neighbors_by_worldpoints=True, use_gpu=True, output_folder=tmp_path, load_segments=True)
    for i in range(inp["V"]):
        _add(L, inp, i, ())
    L.match_images()
    L.reconstruct_3d_lines(3, False)
    a, b = _digest(L), _digest(explicit_run)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert L.stats()["lines3D"] == explicit_run.stats()["lines3D"]
    L.close()


def test_add_image_without_segments_names_the_cache_file(inp, tmp_path):
    w, h = (int(x) for x in inp["wh"][0])
    path = line3d.segment_cache_path(tmp_path, 0, w, h, -1)
    off = line3d.Line3D(neighbors_by_worldpoints=True, use_gpu=True, output_folder=tmp_path, load_segments=False)
    os.makedirs(tmp_path / "L3D++_data")
    line3d.write_segment_cache(path, inp["segs"][0])
    with pytest.raises(capi.L3DError) as e:          # load_segments = false: the file is not read even though it exists
        _add(off, inp, 0, ())
    assert path in str(e.value) and "load_segments" in str(e.value)
    off.close()
    L = line3d.Line3D(neighbors_by_worldpoints=True, use_gpu=True, output_folder=tmp_path, load_segments=True)
    with pytest.raises(capi.L3DError) as e:          # no cache file for this view
        _add(L, inp, 1, ())
    assert line3d.segment_cache_path(tmp_path, 1, *(int(x) for x in inp["wh"][1]), -1) in str(e.value)
    bad = line3d.segment_cache_path(tmp_path, 2, *(int(x) for x in inp["wh"][2]), -1)
    open(bad, "wb").write(open(path, "rb").read()[:100])
    with pytest.raises(capi.L3DError) as e:          # a truncated cache file: its segment count exceeds what is left of it
        _add(L, inp, 2, ())
    assert bad in str(e.value) and "exceed the remaining bytes" in str(e.value)
    _add(L, inp, 0, ())                              # the valid one is accepted
    L.close()


def test_cache_file_name_follows_max_img_width(inp, tmp_path):
    """with max_img_width the cache is looked up under the downscaled size, like the reference names it"""
    w, h = (int(x) for x in inp["wh"][0])
    os.makedirs(tmp_path / "L3D++_data")
    path = line3d.segment_cache_path(tmp_path, 0, w, h, 1000)
    assert "_1000x" in path or "x1000_" in path
    line3d.write_segment_cache(path, inp["segs"][0])
    L = line3d.Line3D(neighbors_by_worldpoints=True, use_gpu=True, output_folder=tmp_path, load_segments=True, max_img_width=1000)
    _add(L, inp, 0, ())
    with pytest.raises(capi.L3DError) as e:
        _add(L, inp, 1, ())
    assert line3d.segment_cache_path(tmp_path, 1, *(int(x) for x in inp["wh"][1]), 1000) in str(e.value)
    L.close()
