"""The calls that take host arrays share one pair of staging buffers per context.  One context runs undistortion, JPEG decoding,
image preparation, remap, undistortion maps, dense matching, triangulation and median depths in host mode, and the line bundling,
the diffusion and the weight argsort, interleaved, with sizes that grow and then shrink; every result must be byte for byte what the
same call gives on a fresh context.  A corrupt JPEG in the sequence must leave its host outputs untouched and the next call right."""
import os

import numpy as np
import pytest

from line3dpp_b200 import capi, synth
from tests import jpeg_model as jm
from tests import nvm_util as nu
from tests import rdd_model as rm
from tests import tri_model as tm
from tests import util
from tests.test_sweep_paths_gpu import argsort_f32, tie_heavy_keys

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden")
K = np.array([[900.0, 0, 500.3], [0, 905.0, 301.7], [0, 0, 1]])
RAD, TAN = (-0.21, 0.05, -0.004), (1.2e-3, -7e-4)


def _pitched(rng, shape, pad):
    """a random uint8 image whose rows are `pad` bytes longer than its width: staged with a pitched copy"""
    full = rng.integers(0, 256, (shape[0], shape[1] + pad) + shape[2:], dtype=np.uint8)
    return full[:, :shape[1]]


def _corrupt_jpeg():
    """a restart-coded file whose scan starts with a run of 1 bits: no Huffman code matches, found on the GPU after the kernels ran"""
    good = jm.build_case(dict(w=40, h=24, sampling="420", restart=2, seed=7))
    k = good.index(b"\xFF\xDA")
    k += 2 + (good[k + 2] << 8 | good[k + 3])
    return good[:k + 4] + b"\xFF\x00" * 8 + good[k + 20:]


def _steps(scene):
    rng = np.random.default_rng(11)
    photos = [open(os.path.join(GOLD, f"jpeg_photo_{i}.jpg"), "rb").read() for i in (0, 1)]
    steps = []

    def undistort(h, w, pad):
        imgs = [_pitched(rng, (h, w, 3), pad), rng.integers(0, 256, (h // 2 + 1, w // 2 + 1, 3), dtype=np.uint8)]
        steps.append(("undistort", lambda c: c.undistort(imgs, K, RAD, TAN)))

    def jpeg(files):
        steps.append(("decode_jpeg_gray", lambda c: c.decode_jpeg_gray(files)))

    def prepare(h, w, pad, max_w):
        imgs = [_pitched(rng, (h, w, 3), pad), rng.integers(0, 256, (h, w | 1), dtype=np.uint8)]
        steps.append(("prepare_gray", lambda c: c.prepare_gray(imgs, max_w)))

    def remap(h, w, oh, ow):
        assert w % 2 == 1      # the maps are staged behind a grey image of odd length
        img = rng.integers(0, 256, (h, w), dtype=np.uint8)
        xy = np.stack([rng.integers(-2, w + 2, (oh, ow)), rng.integers(-2, h + 2, (oh, ow))], 2).astype(np.int16)
        fr = rng.integers(0, 1024, (oh, ow)).astype(np.uint16)
        steps.append(("remap", lambda c: [c.remap(img, xy, fr)]))

    def undistort_map(w, h, size):
        steps.append(("undistort_map", lambda c: c.undistort_map(w, h, K, RAD, TAN, out_size=size)))

    def dense(src, tgt):
        pi = util.pair_inputs(scene, src, tgt)
        steps.append(("match_dense", lambda c: c.match_dense(src, tgt, pi["F"], 0.25, len(pi["ls"]), len(pi["lt"]))))

    def triangulate(n, hi, ncam):
        p = tm.ring_points(n, 3, hi, ncam=ncam, seed=n)
        steps.append(("triangulate_points", lambda c: c.triangulate_points(p.ptr, p.cam, p.xy, p.P)))

    def medians(ncam, n):
        q = tm.join_medians(tm.median_lists(ncam, n_points=n), tm.median_edges())
        steps.append(("median_depths", lambda c: c.median_depths(*q)))

    before, _, opt_ptr, opt_res = nu.load_opt_pairs()
    cams, shift = nu.optimizer_inputs(nu.load_inputs())
    before = before + np.tile(shift, 2)

    def optimize(n, max_iter):
        ptr = opt_ptr[:n + 1]
        res = opt_res[:ptr[-1]]
        steps.append(("optimize_lines", lambda c: c.optimize_lines(before[:n], ptr, res[:, 0].astype(np.int32), res[:, 2:6], cams, max_iter)))

    def optimize_without_residuals(n):
        """res_cam, res_xy and cams are null while num_cams > 0: nothing of them is staged"""
        p, ptr = np.ascontiguousarray(before[:n]), np.zeros(n + 1, np.int64)

        def run(c):
            out, valid, summ = np.zeros((n, 6)), np.zeros(n, np.int32), np.zeros(8)
            c._chk(c.L.l3d_optimize_lines(c.h, n, capi._p(p), capi._p(ptr), None, None, len(cams), None, 10, capi._p(out), capi._p(valid),
                                          capi._p(summ)), "l3d_optimize_lines")
            return out, valid, summ
        steps.append(("optimize_lines without residuals", run))

    def rdd(name):
        graph = rm.BUILDERS[name]()

        def run(c):
            oi, oj, ow, ms = c.rdd(*graph, 10)
            assert ms > 0
            return oi, oj, ow
        steps.append(("rdd", run))

    def argsort(n):
        keys = tie_heavy_keys(n, n)

        def run(c):
            rc, perm = argsort_f32(c, keys)
            assert rc == 0
            return [perm]
        steps.append(("argsort_f32", run))

    # small
    undistort(41, 57, 3); jpeg(photos[:1]); prepare(45, 61, 0, 32); remap(23, 37, 19, 29); undistort_map(57, 41, None); dense(0, 1)
    triangulate(500, 4, 64); medians(20, 500); optimize(40, 250); rdd("tiny"); argsort(257)
    # large
    undistort(1080, 1920, 64); steps.append(("corrupt JPEG", None)); jpeg(photos); prepare(1200, 1600, 5, 1000); remap(1001, 1501, 1100, 1700)
    undistort_map(1920, 1080, (2001, 1203)); dense(2, 3); triangulate(60000, 12, 1500); medians(800, 30000); argsort((1 << 20) + 3); rdd("ladder")
    optimize(len(before), 250)
    # small again, behind staging buffers the large images left
    undistort(17, 29, 0); optimize_without_residuals(30); rdd("hubs"); prepare(33, 47, 2, 0); argsort(4099); remap(9, 13, 11, 15); jpeg(photos[1:])
    undistort_map(31, 17, (20, 40)); dense(5, 1); triangulate(700, 5, 64); medians(10, 400); optimize(7, 3)
    return steps


def _bytes(result):
    return [np.ascontiguousarray(a).tobytes() for a in result]


def test_one_context_through_growing_and_shrinking_host_calls():
    scene = synth.make_scene(8, 700, 11, "dense")
    descs = util.scene_descs(scene)
    steps = _steps(scene)
    bad = _corrupt_jpeg()
    ctx = capi.Context(0)
    try:
        ctx.set_views(descs, scene.segs)
        shared = []
        for name, run in steps:
            if run is None:     # a corrupt file among good ones: the call fails and writes none of its host outputs
                files = [open(os.path.join(GOLD, "jpeg_photo_1.jpg"), "rb").read(), bad]
                outs = [np.full(capi.jpeg_info(f)[::-1], 7, np.uint8) for f in files]
                with pytest.raises(capi.L3DError, match="image 1: corrupt entropy-coded data"):
                    ctx.decode_jpeg_gray(files, out=outs)
                assert all(np.all(o == 7) for o in outs)
                shared.append(None)
            else:
                shared.append(_bytes(run(ctx)))
    finally:
        ctx.close()
    for (name, run), got in zip(steps, shared):
        if run is None:
            continue
        fresh = capi.Context(0)
        try:
            if name == "match_dense":
                fresh.set_views(descs, scene.segs)
            assert got == _bytes(run(fresh)), name
        finally:
            fresh.close()
