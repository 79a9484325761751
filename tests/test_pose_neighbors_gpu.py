"""l3d_pose_neighbors on the GPU against the float64 model (tests/pose_model.py): n_i, every nonzero common(i, j) and every neighbour list
exactly; the neighbours feed Line3D as the model's virtual world points would; every rejection with its message."""
import numpy as np
import pytest

from line3dpp_b200 import capi, line3d, synth
from tests import pose_model as pm
from tests.test_pose_model_cpu import SCENES, coincident_scene, shifted_pair_scene

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


def descs(V):
    return capi.make_pose_views(V.cam_ids, V.K, V.R, V.t, V.width, V.height, V.depth)


def check_exact(ctx, V, gx, gy, nn_list=(1, 3, 10)):
    d = descs(V)
    n_dev, ijc = ctx.pose_covisibility(d, gx, gy)
    n, cm = pm.counts(V, gx, gy)
    np.testing.assert_array_equal(n_dev, n)
    i, j = np.nonzero(cm)
    want = np.stack([i, j, cm[i, j]], axis=1)
    np.testing.assert_array_equal(ijc, want)
    for nn in nn_list:
        got, n2, _ = ctx.pose_neighbors(d, nn, gx, gy)
        np.testing.assert_array_equal(n2, n)
        assert [list(map(int, g)) for g in got] == pm.select(V, n, cm, nn), nn


EXACT = {
    **{k: (v[0], v[1], v[2]) for k, v in SCENES.items()},
    "ring_67_tiles": (lambda: pm.ring(67, seed=4), 7, 5),
    "grid_12x9": (lambda: pm.grid_survey(12, 9, seed=3), 9, 7),
    "random_40": (lambda: pm.random_poses(40, seed=11), 11, 3),
    "random_behind": (lambda: pm.random_poses(30, seed=12, spread=0.8), 6, 6),
    "borders": (lambda: shifted_pair_scene([0.0, 1.0, 2.0, 2.5, 3.0, 4.0, 5.0, 0.5]), 5, 1),
    "borders_2d": (lambda: shifted_pair_scene([0.0, 1.0, 3.0, 4.0], gx=10, gy=2), 10, 2),
    "coincident": (coincident_scene, 8, 6),
    "one_view": (lambda: pm.ring(1), 4, 3),
    "two_views": (lambda: pm.ring(2, radius=1.0), 8, 8),
    "two_views_close": (lambda: pm.ring(40, radius=4.0).subset([0, 1]), 8, 8),
}


@pytest.mark.parametrize("scene", sorted(EXACT))
def test_exact_counts_and_neighbors(ctx, scene):
    make, gx, gy = EXACT[scene]
    check_exact(ctx, make(), gx, gy)


@pytest.mark.parametrize("gx,gy", [(1, 1), (2, 1), (1, 3), (5, 7), (13, 11), (32, 24), (64, 64), (4096, 1)])
def test_grid_sizes(ctx, gx, gy):
    check_exact(ctx, pm.ring(9, seed=gx + gy), gx, gy, nn_list=(2, 10))


def test_large_scene_on_a_subset():
    """2400 views (a ring of 1200 and a 40 x 30 grid survey, far apart), checked on 40 random views"""
    A = pm.ring(1200, radius=40.0, depth=40.0, seed=7)
    B = pm.grid_survey(40, 30, spacing=2.0, seed=8)
    B.t = B.t - B.R @ np.array([500.0, 0.0, 0.0])     # the survey 500 units along x
    V = pm.Views(np.concatenate([A.cam_ids, B.cam_ids + 5000]), np.concatenate([A.K, B.K]), np.concatenate([A.R, B.R]),
                 np.concatenate([A.t, B.t]), np.concatenate([A.width, B.width]), np.concatenate([A.height, B.height]),
                 np.concatenate([A.depth, B.depth]))
    gx, gy = 4, 3
    sub = sorted(np.random.default_rng(1).choice(len(V), 40, replace=False).tolist())
    c = capi.Context(0)
    try:
        d = descs(V)
        n_dev, ijc = c.pose_covisibility(d, gx, gy)
        got, _, _ = c.pose_neighbors(d, 10, gx, gy)
    finally:
        c.close()
    n, cm = pm.counts(V, gx, gy, sub)
    np.testing.assert_array_equal(n_dev, n)
    for k, i in enumerate(sub):
        rows = ijc[ijc[:, 0] == i]
        j = np.flatnonzero(cm[k])
        np.testing.assert_array_equal(rows[:, 1], j)
        np.testing.assert_array_equal(rows[:, 2], cm[k, j])
    assert [list(map(int, got[i])) for i in sub] == pm.select(V, n, cm, 10, sub)
    assert sum(len(g) for g in got) > 20000


def test_line3d_end_to_end():
    """Line3D with the model's virtual world points and Line3D with pose_neighbors' lists match the same view pairs and reconstruct the
    same 3D lines, byte for byte"""
    sc = synth.make_scene(12, 150, 5, "ring2")
    V = pm.Views(sc.cam_ids, sc.K, sc.R, sc.t, sc.width, sc.height, sc.median_depth.astype(np.float64))
    gx, gy = 16, 12
    wps = pm.world_point_lists(V, gx, gy)
    nb = line3d.pose_neighbors(sc.cam_ids, sc.K, sc.R, sc.t, sc.width, sc.height, sc.median_depth, num_neighbors=10, gx=gx, gy=gy)
    assert [list(map(int, x)) for x in nb] == pm.pose_neighbors(V, gx, gy, 10)
    out = []
    for by_wps, lists in ((True, wps), (False, nb)):
        L = line3d.Line3D(neighbors_by_worldpoints=by_wps)
        for i in range(sc.num_views):
            L.add_image(sc.cam_ids[i], sc.width, sc.height, sc.K[i], sc.R[i], sc.t[i], sc.median_depth[i], lists[i], sc.segs[i])
        L.match_images(num_neighbors=10)
        L.reconstruct_3d_lines(3, True)
        out.append((L.pairs(), L.segments3d(), L.residuals()))
        L.close()
    (pa, sa, ra), (pb, sb, rb) = out
    assert len(pa) > 12 and len(sa) > 20
    np.testing.assert_array_equal(pa, pb)
    assert sa.tobytes() == sb.tobytes() and ra.tobytes() == rb.tobytes()


def _bad(V, i, **kw):
    d = descs(V)
    for k, v in kw.items():
        if k in ("R", "t"):
            getattr(d[i], k)[0] = v
        else:
            setattr(d[i], k, v)
    return d


@pytest.mark.parametrize("field,value,msg", [
    ("median_depth", 0.0, "median_depth must be finite and > 0"), ("median_depth", -1.0, "median_depth must be finite and > 0"),
    ("median_depth", float("inf"), "median_depth must be finite and > 0"), ("median_depth", float("nan"), "median_depth must be finite and > 0"),
    ("width", 0, "width and height must be at least 1"), ("height", -3, "width and height must be at least 1"),
    ("fx", 0.0, "fx or fy is zero or not finite"), ("fy", float("nan"), "fx or fy is zero or not finite"), ("fx", float("inf"), "fx or fy is zero or not finite"),
    ("R", float("nan"), "R is not finite"), ("t", float("inf"), "t is not finite"), ("cam_id", 5, "duplicate camID, already view 1"),
])
def test_rejections(ctx, field, value, msg):
    V = pm.ring(6, cam_ids=[3, 5, 8, 13, 21, 34])
    d = _bad(V, 4, **{field: value})
    cam = 5 if field == "cam_id" else 21
    for call in (lambda: ctx.pose_neighbors(d, 10), lambda: ctx.pose_covisibility(d)):
        with pytest.raises(capi.L3DError, match=rf"\(-1\): l3d_pose_\w+: view 4 \(camID {cam}\): {msg}"):
            call()


@pytest.mark.parametrize("gx,gy", [(0, 4), (4, 0), (-1, 1)])
def test_rejected_grid(ctx, gx, gy):
    with pytest.raises(capi.L3DError, match=r"\(-1\): l3d_pose_neighbors: gx and gy must be at least 1"):
        ctx.pose_neighbors(descs(pm.ring(3)), 10, gx, gy)


def test_too_many_points(ctx):
    with pytest.raises(capi.L3DError, match=r"\(-4\): .*L3D_POSE_MAX_POINTS"):
        ctx.pose_neighbors(descs(pm.ring(5)), 10, 4096, 4096)


def test_python_entry_names_the_view():
    V = pm.ring(3)
    with pytest.raises(capi.L3DError, match=r"view 1 \(camID 1\): median_depth"):
        line3d.pose_neighbors(V.cam_ids, V.K, V.R, V.t, 640, 480, [4.0, 0.0, 4.0])
