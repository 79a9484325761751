"""The row windows k_row_windows writes before k_match_topk scans (l3d_match.cuh, read back with l3d_match_row_windows) against the numpy
model of the level-1 pre-filter (tests/level1_model.py) on the device's own pencil basis and sorted table: the pencil parameters of both
float epipolar lines, the flag of rows outside the pencil model, and per arc class the two window ends as np.searchsorted finds them.
An off-by-one at a window edge changes which targets a row scans, but the target at the edge rarely matches, so the match lists alone
would not show it."""
import numpy as np
import pytest

from line3dpp_b200 import synth
from tests import level1_model as m
from tests import util

pytestmark = pytest.mark.gpu


def _kappa(u, v, e):
    """(kappa, off, kappa in units before rounding) of a float line; a non-finite angle is kappa 0 and off, as on the device"""
    x, y, z = m.S * float(e[0]), m.S * float(e[1]), float(e[2])
    k = np.arctan2(x * v[0] + y * v[1] + z * v[2], x * u[0] + y * u[1] + z * u[2])
    if not np.isfinite(k):
        return 0, True, 0.0
    kappa, off = m.line_kappa(u, v, e)
    return kappa, off, k * m.TU


def check_pair(ctx, pair, F, src, nt):
    """every row of `pair` (source segments src, float F, nt target segments) against the model; returns counts of the cases met"""
    win, (u, v), off, starts = ctx.row_windows(pair, len(src), nt)
    assert off[0] == 0 and off[-1] == nt and (np.diff(off) >= 0).all()
    for c in range(m.NCLS):
        assert (np.diff(starts[off[c]:off[c + 1]].astype(np.int64)) >= 0).all(), c      # a class is sorted by arc start
    seen = dict(rows=len(src), rall=0, kb_max=0, wrap=0, half=0)
    for r, s in enumerate(src):
        w = [int(x) for x in win[r]]
        ks, rall = [], False
        for i, (x, y) in enumerate(((s[0], s[1]), (s[2], s[3]))):
            k, o, raw = _kappa(u, v, m.epipolar_line(F, x, y))
            if w[i] != k:
                # numpy's and CUDA's atan2 may differ in the last bit: only a kappa that lies on a rounding half may round apart
                assert (w[i] - k) & m.M32 in (1, m.M32) and abs(raw - np.floor(raw) - 0.5) < 1e-4, (pair, r, i, w[i], k, raw)
                seen["half"] += 1
                k = w[i]
            ks.append(k)
            rall |= o
        assert w[2] == int(rall) and w[3] == 0, (pair, r, w[:4], rall)
        k1, k2 = ks
        ka, kb = (k1, k2) if ((k2 - k1) & m.M32) < 0x80000000 else (k2, k1)
        seen["rall"] += rall
        seen["kb_max"] += kb == m.M32 and not rall
        for c in range(m.NCLS):
            lo, hi = int(off[c]), int(off[c + 1])
            cls = starts[lo:hi]
            key = (ka - (1 << (m.CLS0 + c))) & m.M32
            if rall:
                want = (lo, lo)
            else:
                want = (lo + int(np.searchsorted(cls, np.uint32(key), "left")),
                        hi if kb == m.M32 else lo + int(np.searchsorted(cls, np.uint32(kb + 1), "left")))
                seen["wrap"] += key > kb and hi > lo
            assert (w[4 + 2 * c], w[5 + 2 * c]) == want, (pair, r, c, (w[4 + 2 * c], w[5 + 2 * c]), want, ka, kb)
    assert seen["half"] <= max(2, len(src) // 1000)
    return seen, off


def test_bench_geometry_and_a_pair_range(gpu_ctx):
    """the benchmark's geometry (ring +-5, 3000 segments per view): whole calls and a range of the pair list, rows counted from its first pair"""
    sc = synth.make_scene(8, 3000, 1004, "ring5")
    gpu_ctx.set_views(util.scene_descs(sc), sc.segs)
    pairs = synth.view_pairs(sc.neighbors)
    F = util.pair_F(sc, pairs)
    gpu_ctx.match_pairs(pairs, F, 0.25, 10)
    for p in (0, 7):
        check_pair(gpu_ctx, p, F[p], sc.segs[pairs[p][0]], len(sc.segs[pairs[p][1]]))
    gpu_ctx.match_pairs_range(pairs, F, 5, 9, 0.25, 10)
    for p in (5, 8):
        check_pair(gpu_ctx, p, F[p], sc.segs[pairs[p][0]], len(sc.segs[pairs[p][1]]))


def crafted_scene():
    """the "forward" pair with source rows whose epipolar lines lie at kappa ~ 0 (windows that wrap, kb = 2^32 - 1) and rows through the
    source epipole (F*p is rounding noise: the row skips level 1)"""
    sc = util.two_view_scene("forward", 1500, 31)
    F = util.pair_F(sc, [(0, 1)])[0]
    u, v, _ = m.basis(F)
    L = F.astype(np.float64).reshape(3, 3).T @ np.array([m.S * v[0], m.S * v[1], v[2]])    # source points whose line has kappa 0
    rng = np.random.default_rng(3)
    y = rng.uniform(100, 2100, (1500, 2))
    x = -(L[1] * y + L[2]) / L[0]
    on_line = np.stack([x[:, 0], y[:, 0], x[:, 1], y[:, 1]], 1)
    e = np.linalg.svd(F.astype(np.float64).reshape(3, 3))[2][-1]
    ex, ey = e[0] / e[2], e[1] / e[2]
    a = np.linspace(0, np.pi, 40, endpoint=False)
    through = np.stack([np.full_like(a, ex), np.full_like(a, ey), ex + 150 * np.cos(a), ey + 150 * np.sin(a)], 1)
    sc.segs[0] = np.ascontiguousarray(np.concatenate([sc.segs[0], on_line, through]).astype(np.float32))
    return sc


@pytest.mark.parametrize("f64", [False, True], ids=["ref_gpu", "ref_cpu"])
def test_wrapping_windows_the_last_kappa_and_rows_off_the_pencil(gpu_ctx, f64):
    """REF_CPU semantics (double F; the windows come from its float copy, as the kernel's float filter does) reads the same windows"""
    sc = crafted_scene()
    gpu_ctx.set_views(util.scene_descs(sc), sc.segs)
    pairs = np.array([(0, 1)], np.int32)
    F = util.pair_F(sc, pairs)
    if f64:
        Fd = np.array([synth.fundamental(sc.K[0], sc.R[0], sc.t[0], sc.K[1], sc.R[1], sc.t[1]).reshape(9)])
        gpu_ctx.match_pairs_f64(pairs, Fd, 0.25, 10)
        F = Fd.astype(np.float32)
    else:
        gpu_ctx.match_pairs(pairs, F, 0.25, 10)
    seen, off = check_pair(gpu_ctx, 0, F[0], sc.segs[0], len(sc.segs[1]))
    assert seen["rall"] > 0 and seen["kb_max"] > 0 and seen["wrap"] > 100, seen
    assert off[-2] < off[-1]                                    # the wide class: targets through the epipole


def test_target_view_beyond_the_ring_and_the_staged_starts(gpu_ctx):
    """target views of several TMA passes (> 3072 segments), one of them with more arc starts than k_row_windows stages (> 12000):
    that pair's windows are searched in the table itself"""
    sc = synth.make_scene(4, 3600, 17, "dense")
    sc.segs[0] = sc.segs[0][:300].copy()
    sc.segs[3] = np.ascontiguousarray(np.concatenate([sc.segs[3], sc.segs[2], sc.segs[1], sc.segs[2]]))
    gpu_ctx.set_views(util.scene_descs(sc), sc.segs)
    pairs = np.array([(0, 1), (0, 3)], np.int32)
    F = util.pair_F(sc, pairs)
    gpu_ctx.match_pairs(pairs, F, 0.25, 10)
    for p, (s, t) in enumerate(pairs):
        _, off = check_pair(gpu_ctx, p, F[p], sc.segs[s], len(sc.segs[t]))
        assert t != 3 or off[m.NCLS] > 12000


def test_level1_off(gpu_ctx):
    """epi_overlap < 0.01: every target is in the wide class, every window of classes 0 .. 7 is empty; the kappas are still the rows'"""
    sc = synth.make_scene(3, 700, 11, "dense")
    gpu_ctx.set_views(util.scene_descs(sc), sc.segs)
    pairs = np.array([(0, 1), (2, 0)], np.int32)
    F = util.pair_F(sc, pairs)
    gpu_ctx.match_pairs(pairs, F, 0.005, 10)
    for p, (s, t) in enumerate(pairs):
        _, off = check_pair(gpu_ctx, p, F[p], sc.segs[s], len(sc.segs[t]))
        assert (off[:m.NCLS + 1] == 0).all()
