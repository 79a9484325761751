"""The model of l3d_pose_neighbors (tests/pose_model.py) against a loop-and-set restatement of findVisualNeighborsFromWPs fed the model's
virtual world points, on scenes that reach every branch of the selection; and the Python mirror of l3d_pose_view.  No GPU needed."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from line3dpp_b200 import capi
from tests import pose_model as pm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def shifted_pair_scene(shifts, gx=5, gy=1):
    """identical nadir-free cameras (R = I, f = 500, 500 x 100 px, depth 5) translated along x by `shifts` world units: 100 px per unit,
    so samples fall exactly on pixel 0 and on the width"""
    K = pm.intrinsics(500.0, 500, 100)
    ts = [np.array([-s, 0.0, 0.0]) for s in shifts]
    n = len(shifts)
    return pm.Views(np.arange(n), np.repeat(K[None], n, 0), np.repeat(np.eye(3)[None], n, 0), ts, 500, 100, 5.0)


def with_extra(V, K, R, t, w, h, depth, cam):
    return pm.Views(np.append(V.cam_ids, cam), np.concatenate([V.K, K[None]]), np.concatenate([V.R, R[None]]), np.concatenate([V.t, t[None]]),
                    np.append(V.width, w), np.append(V.height, h), np.append(V.depth, depth))


def coincident_scene():
    """a ring plus views at the centre of view 0 (baseline 0), turned a little, and one far away looking away from everything"""
    V = pm.ring(10, jitter=0.0, cam_ids=np.arange(10) * 3)
    C0 = -V.R[0].T @ V.t[0]
    for k, ang in enumerate((0.05, -0.05)):
        c, s = np.cos(ang), np.sin(ang)
        R = V.R[0] @ np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])
        V = with_extra(V, V.K[0], R, -R @ C0, 640, 480, 4.0, 100 + k)
    R, t = pm.look_at([0.0, 50.0, 0.0], [0.0, 100.0, 0.0], up=(1.0, 0.0, 0.0))
    return with_extra(V, V.K[0], R, t, 640, 480, 4.0, 7)


SCENES = {
    "ring_ties": (lambda: pm.ring(12, jitter=0.0, cam_ids=[11, 3, 7, 0, 5, 9, 1, 10, 2, 8, 4, 6]), 8, 6),
    "ring": (lambda: pm.ring(16, seed=2), 10, 8),
    "grid": (lambda: pm.grid_survey(6, 5, seed=1), 8, 6),
    "random": (lambda: pm.random_poses(20, seed=5), 6, 5),
    "shifted": (lambda: shifted_pair_scene([0.0, 2.5, 30.0, 33.0]), 5, 1),
    "coincident": (coincident_scene, 8, 6),
}


@pytest.mark.parametrize("num_neighbors", [1, 2, 3, 5, 10, 64])
@pytest.mark.parametrize("scene", sorted(SCENES))
def test_model_matches_the_reference_loop(scene, num_neighbors):
    make, gx, gy = SCENES[scene]
    V = make()
    want = pm.reference_neighbors(V, pm.world_point_lists(V, gx, gy), num_neighbors)
    assert pm.pose_neighbors(V, gx, gy, num_neighbors) == want


def _candidates(V, gx, gy):
    """per view: [(common, score, axis)] of every co-visible view, and n"""
    n, cm = pm.counts(V, gx, gy)
    cams = pm.cams_of(V)
    return n, cm, [[(int(cm[i, j]), pm.score(cm[i, j], n[i], n[j]), pm.axis_angle(cams[i], cams[j])) for j in range(len(V)) if cm[i, j]]
                   for i in range(len(V))]


def test_scenes_reach_every_branch():
    # score ties among candidates
    V = SCENES["ring_ties"][0]()
    _, _, c = _candidates(V, 8, 6)
    assert any(len({s for cc, s, a in row if cc > 4}) < len([1 for cc, s, a in row if cc > 4]) for row in c)
    # views facing away: co-visible with more than 4 common points but past the axis gate
    assert any(cc > 4 and a >= np.float32(1.571) for row in c for cc, s, a in row)
    # the 0.8 cut active (more candidates than neighbours, some below 0.8 x best) and inactive (fewer)
    V = SCENES["random"][0]()
    _, _, c = _candidates(V, 6, 5)
    gated = [[(cc, s) for cc, s, a in row if cc > 4 and a < np.float32(1.571)] for row in c]
    assert any(len(g) > 3 and min(s for _, s in g) <= np.float32(0.8) * max(s for _, s in g) for g in gated)
    assert any(0 < len(g) < 64 for g in gated)
    # common exactly 4 and 5 (samples exactly on pixel 0 and on the width)
    V = SCENES["shifted"][0]()
    n, cm = pm.counts(V, 5, 1)
    assert cm[0, 1] == 5 and cm[2, 3] == 4, cm
    # coincident centres: baseline 0, so the gate rejects them while other neighbours are already in use; the far view sees nobody
    V = coincident_scene()
    n, cm = pm.counts(V, 8, 6)
    cams = pm.cams_of(V)
    assert cm[0, 10] > 4 and cm[0, 11] > 4 and pm.baseline(cams[0], cams[10]) == 0
    nb = pm.pose_neighbors(V, 8, 6, 5)
    assert 100 not in nb[0] and 101 not in nb[0] and len(nb[0]) > 1
    assert cm[12].sum() == 0 and nb[12] == []


def test_sample_order_and_back_projection():
    """sample s = r * gx + c of view i is point i * G + s at ((c + 0.5) w / gx, (r + 0.5) h / gy) and depth median_depth"""
    V = pm.random_poses(3, seed=9)
    gx, gy = 7, 4
    X = pm.sample_points(V, gx, gy)
    for i in range(3):
        for s in (0, 5, 27):
            c, r = s % gx, s // gx
            q = V.R[i] @ X[i * gx * gy + s] + V.t[i]
            p = V.K[i] @ q
            assert q[2] == pytest.approx(V.depth[i], rel=1e-12)
            assert p[0] / p[2] == pytest.approx((c + 0.5) * V.width[i] / gx, rel=1e-9)
            assert p[1] / p[2] == pytest.approx((r + 0.5) * V.height[i] / gy, rel=1e-9)


def test_pose_view_mirror_matches_the_header(tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no gcc")
    fields = [n for n, _ in capi.PoseView._fields_]
    src = tmp_path / "pose.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "l3d_capi.h"\nint main(void)\n{\n'
                   + 'printf("%zu\\n", sizeof(l3d_pose_view));\n'
                   + "".join(f'printf("%zu\\n", offsetof(l3d_pose_view, {f}));\n' for f in fields) + "return 0;\n}\n")
    exe = tmp_path / "pose"
    subprocess.run([gcc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(x) for x in subprocess.check_output([str(exe)], text=True).split()]
    assert got == [ctypes.sizeof(capi.PoseView)] + [getattr(capi.PoseView, f).offset for f in fields]
