"""Tie-point triangulation and median depths on the GPU (l3d_triangulate_points, l3d_median_depths, DESIGN.md §6b) against numpy, the
Pix4D reader against a numpy restatement of main_pix4d.cpp, and every new reader end to end: reader -> addImage -> matchImages ->
reconstruct3Dlines equals the same run fed with the scene's own cameras, bit for bit."""
import numpy as np
import pytest

from line3dpp_b200 import capi, line3d
from tests import sfm_scene as ss

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = capi.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def scene():
    return ss.Scene()


def _look_at(C):
    z = -C / np.linalg.norm(C)
    x = np.cross([0.0, 0.0, 1.0], z); x /= np.linalg.norm(x)
    return np.stack([x, np.cross(z, x), z])


def _random_problem(n, lo, hi, ncam=64, seed=0, noise=0.5):
    """n points in [-5, 5]^3 seen by lo..hi of ncam cameras on a ring of radius 30 (f = 1200 px), N(0, noise px) on every observation"""
    rng = np.random.default_rng(seed)
    K = np.array([[1200.0, 0, 960], [0, 1200.0, 540], [0, 0, 1]])
    ang = np.linspace(0, 2 * np.pi, ncam, endpoint=False)
    Cs = np.stack([30 * np.cos(ang), 30 * np.sin(ang), 10 + 2 * np.sin(3 * ang)], 1)
    P = np.stack([K @ np.hstack([_look_at(C), (-_look_at(C) @ C)[:, None]]) for C in Cs])
    X = rng.uniform(-5, 5, (n, 3))
    cnt = rng.integers(lo, hi + 1, n)
    ptr = np.zeros(n + 1, np.int64); ptr[1:] = np.cumsum(cnt)
    cam = np.concatenate([rng.choice(ncam, c, replace=False) for c in cnt]).astype(np.int32)
    h = np.einsum("nij,nj->ni", P[cam], np.hstack([np.repeat(X, cnt, 0), np.ones((int(ptr[-1]), 1))]))
    xy = h[:, :2] / h[:, 2:] + rng.normal(0, noise, (int(ptr[-1]), 2))
    return ptr, cam, xy, P, Cs


def _numpy_triangulation(ptr, cam, xy, P):
    """A^T A built in numpy, eigh: X, valid, kappa = lambda_max / (lambda_2 - lambda_1)"""
    Pc = P[cam]
    r1 = -Pc[:, 1] + xy[:, 1:2] * Pc[:, 2]; r2 = Pc[:, 0] - xy[:, 0:1] * Pc[:, 2]
    outer = np.einsum("ni,nj->nij", r1, r1) + np.einsum("ni,nj->nij", r2, r2)
    seg = np.repeat(np.arange(len(ptr) - 1), np.diff(ptr))
    A = np.zeros((len(ptr) - 1, 4, 4)); np.add.at(A, seg, outer)
    w, V = np.linalg.eigh(A)
    v = V[:, :, 0]
    with np.errstate(divide="ignore", invalid="ignore"):
        X = v[:, :3] / v[:, 3:]
        nrm = np.sqrt(X[:, 0] * X[:, 0] + X[:, 1] * X[:, 1] + X[:, 2] * X[:, 2])
        kappa = w[:, 3] / (w[:, 1] - w[:, 0])
    valid = ((np.diff(ptr) >= 3) & (nrm > 1e-12)).astype(np.int32)
    X[np.diff(ptr) < 3] = 0
    return X, valid, kappa


def test_triangulation_against_numpy(ctx):
    """10^5 points with 3-20 noisy observations: X to 1e-9 relative wherever kappa = lambda_max / (lambda_2 - lambda_1) of A^T A is at
    most 1e6 (every point of this scene), the same valid flag everywhere"""
    ptr, cam, xy, P, _ = _random_problem(100000, 3, 20)
    X, valid = ctx.triangulate_points(ptr, cam, xy, P)
    Xn, vn, kappa = _numpy_triangulation(ptr, cam, xy, P)
    assert np.array_equal(valid, vn) and valid.all()
    good = kappa <= 1e6
    assert good.mean() > 0.99
    rel = np.linalg.norm(X - Xn, axis=1) / np.linalg.norm(Xn, axis=1)
    assert rel[good].max() < 1e-9, rel[good].max()


def test_triangulation_degenerate_cases(ctx):
    ptr, cam, xy, P, Cs = _random_problem(8, 3, 3, ncam=16, seed=4, noise=0.0)
    obs = []                                                     # (camera list, xy list) per case
    proj = lambda c, Xh: (P[c] @ Xh)[:2] / (P[c] @ Xh)[2]
    obs.append(([0, 1], [proj(0, np.array([1, 2, 3, 1.0])), proj(1, np.array([1, 2, 3, 1.0]))]))         # 2 observations: invalid
    obs.append(([], []))                                                                                 # none
    d = np.array([0.3, -0.2, 0.05]); d /= np.linalg.norm(d)
    obs.append(([0, 3, 5, 9], [proj(c, np.append(d, 0.0)) for c in (0, 3, 5, 9)]))                      # a point at infinity (w = 0)
    X0 = np.array([0.5, 0.25, -1.0])
    obs.append(([2, 2, 2], [proj(2, np.append(X0, 1.0))] * 3))                                          # coincident observations
    # cameras on a line through the point: three camera centres on one ray from X0
    Kc = np.array([[1200.0, 0, 960], [0, 1200.0, 540], [0, 0, 1]])
    ray = np.array([1.0, 2.0, 0.5]) / np.linalg.norm([1.0, 2.0, 0.5])
    Pl = [Kc @ np.hstack([_look_at(X0 + s * ray), (-_look_at(X0 + s * ray) @ (X0 + s * ray))[:, None]]) for s in (10.0, 20.0, 40.0)]
    Pall = np.concatenate([P, np.stack(Pl)])
    lc = [len(P), len(P) + 1, len(P) + 2]
    obs.append((lc, [(Pall[c] @ np.append(X0, 1.0))[:2] / (Pall[c] @ np.append(X0, 1.0))[2] for c in lc]))
    obs.append(([0, 1, 4], [proj(c, np.array([2.0, -1.0, 0.5, 1.0])) for c in (0, 1, 4)]))             # a regular point
    cnt = [len(o[0]) for o in obs]
    p = np.zeros(len(obs) + 1, np.int64); p[1:] = np.cumsum(cnt)
    c = np.array(sum((o[0] for o in obs), []), np.int32)
    x = np.array(sum((o[1] for o in obs), []), np.float64).reshape(-1, 2)
    X, valid = ctx.triangulate_points(p, c, x, Pall)
    Xn, vn, _ = _numpy_triangulation(p, c, x, Pall)
    assert np.array_equal(valid, vn), (valid, vn)
    assert valid.tolist()[:2] == [0, 0] and not X[:2].any()
    assert valid[2] == 1 and np.linalg.norm(X[2]) > 1e6                                                  # far along d
    np.testing.assert_allclose(X[-1], [2.0, -1.0, 0.5], rtol=0, atol=1e-9)
    # device addresses, asynchronous: the same result
    import torch
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    dp, dc, dx, dP = t(p), t(c), t(x), t(Pall.reshape(-1, 12))
    dX, dv = torch.zeros((len(obs), 3), dtype=torch.float64, device="cuda"), torch.zeros(len(obs), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ctx.triangulate_points_device(len(obs), dp.data_ptr(), dc.data_ptr(), dx.data_ptr(), len(Pall), dP.data_ptr(), dX.data_ptr(), dv.data_ptr())
    ctx.sync()
    assert np.array_equal(dX.cpu().numpy(), X) and np.array_equal(dv.cpu().numpy(), valid)


def test_triangulation_without_shared_memory_staging(ctx):
    """more cameras than fit in shared memory: the matrices are read from global memory, same results"""
    ptr, cam, xy, P, _ = _random_problem(5000, 3, 12, ncam=1500, seed=7)
    X, valid = ctx.triangulate_points(ptr, cam, xy, P)
    Xn, vn, kappa = _numpy_triangulation(ptr, cam, xy, P)
    assert np.array_equal(valid, vn)
    rel = np.linalg.norm(X - Xn, axis=1) / np.linalg.norm(Xn, axis=1)
    assert rel[kappa <= 1e6].max() < 1e-9


def test_triangulation_rejects_bad_host_input(ctx):
    with pytest.raises(capi.L3DError, match="unknown camera"):
        ctx.triangulate_points([0, 3], [0, 1, 5], np.zeros((3, 2)), np.zeros((2, 3, 4)))
    with pytest.raises(capi.L3DError, match="must not decrease"):
        p = np.array([0, 2, 1, 3], np.int64)
        X = np.zeros((3, 3)); v = np.zeros(3, np.int32)
        ctx._chk(ctx.L.l3d_triangulate_points(ctx.h, capi.C.c_longlong(3), capi._p(p), capi._p(np.zeros(3, np.int32)), capi._p(np.zeros(6)), 1,
                                              capi._p(np.zeros(12)), capi._p(X), capi._p(v), 0), "l3d_triangulate_points")


def test_median_depths_exact(ctx):
    rng = np.random.default_rng(9)
    n, nc = 20000, 300
    X = rng.uniform(-50, 50, (n, 3)); valid = (rng.uniform(size=n) > 0.2).astype(np.int32)
    X[5] = [np.inf, 0, 0]; valid[5] = 1                                       # +-Inf is valid: depth inf
    Cs = rng.uniform(-10, 10, (nc, 3))
    sizes = rng.integers(0, 400, nc); sizes[:3] = [0, 1, 5000]
    lptr = np.zeros(nc + 1, np.int64); lptr[1:] = np.cumsum(sizes)
    lpts = rng.integers(0, n, int(lptr[-1])).astype(np.int32)               # repeats included
    lpts[lptr[2]:lptr[2] + 10] = 5
    cnt, med = ctx.median_depths(lptr, lpts, X, valid, Cs)
    for c in range(nc):
        ids = lpts[lptr[c]:lptr[c + 1]]
        ids = ids[valid[ids] != 0]
        d = X[ids] - Cs[c]
        dep = np.sort(np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]).astype(np.float32))
        assert cnt[c] == len(dep)
        assert med[c] == (dep[len(dep) // 2] if len(dep) else np.float32(0)), c


# ---------------------------------------------------------------------------------------------- Pix4D
def _pix4d_centre(scene, i):
    R, t = scene.R[i], scene.t[i]
    return np.array([(R[0][k] * -t[0] + R[1][k] * -t[1]) + R[2][k] * -t[2] for k in range(3)])


def _pix4d_restated(scene, tp_text):
    """main_pix4d.cpp:282-418 in numpy on the text of a tp_pix4d.txt: key images looked up in a map that yields camera 0 for an unknown
    name, feature ids numbered in first-seen order, per key image the list of its observations, the points triangulated by eigh and the
    float median depth over the valid points of each camera: {camera: (list, median or None)}"""
    img2pos = {f"img{i}": i for i in range(scene.V)}
    feats, fobs, per_key, key, pos = {}, [], {}, None, 0
    for line in tp_text.split("\n"):
        tok = line.split()
        if not tok or len(tok[0]) < 2:
            break
        if tok[0].startswith("-"):
            continue
        if len(tok) == 1:
            key, pos = tok[0], img2pos.get(tok[0], 0)
            continue
        f = feats.setdefault(tok[0], len(feats))
        if f == len(fobs):
            fobs.append([])
        fobs[f].append((pos, float(tok[1]), float(tok[2])))
        per_key.setdefault(key, []).append(f)
    P = np.stack([ss.pix4d_P(scene.K[i], scene.R[i], scene.C[i]) for i in range(scene.V)])
    X, valid = ss.triangulate_restated(fobs, P)
    out = {}
    for i in range(scene.V):
        lst = per_key.get(f"img{i}", [])
        C = _pix4d_centre(scene, i)
        d = [np.float32(np.linalg.norm(X[f] - C)) for f in lst if valid[f]]
        out[i] = (lst, np.sort(np.array(d, np.float32))[len(d) // 2] if len(d) > 2 else None)
    return out


def _check_pix4d(scene, folder):
    cams = line3d.read_pix4d(folder, "proj")
    exp = _pix4d_restated(scene, (folder / "proj_tp_pix4d.txt").read_text())
    keep = [i for i in range(scene.V) if exp[i][1] is not None]
    assert [c["id"] for c in cams] == keep
    for c in cams:
        i = c["id"]
        assert c["image"] == f"img{i}.JPG"
        assert np.array_equal(c["K"], scene.K[i]) and np.array_equal(c["R"], scene.R[i]) and np.array_equal(c["t"], scene.t[i])
        # C = R^T (-t) as main_pix4d.cpp:391-392 forms it: the stored centre up to how far the quantised R is from orthonormal
        assert np.array_equal(c["C"], _pix4d_centre(scene, i))
        np.testing.assert_allclose(c["C"], scene.C[i], rtol=0, atol=1e-3)
        assert np.array_equal(c["radial"], scene.radial[i]) and np.array_equal(c["tangential"], scene.tangential[i])
        assert c["worldpoints"].tolist() == exp[i][0]
        assert abs(c["median_depth"] - exp[i][1]) <= 1e-6 * exp[i][1], (i, c["median_depth"], exp[i][1])
    return cams


def test_pix4d_reader(scene, tmp_path):
    scene.write_pix4d(tmp_path)
    assert len(_check_pix4d(scene, tmp_path)) >= 6


def _obs_line(fid, x, y):
    return f"{fid} {ss.num(x)} {ss.num(y)} 1"


def test_pix4d_unknown_key_image_is_camera_0(scene, tmp_path):
    """observations under a key image the camera file does not name are triangulated with camera 0's matrix (std::map::operator[]):
    three points seen twice that way and once by img1 land where camera 0 and camera 1 see them"""
    scene.write_pix4d(tmp_path)
    tp = tmp_path / "proj_tp_pix4d.txt"
    js = [j for j in range(len(scene.X)) if {0, 1} <= {c for c, _, _ in scene.obs[j]}][:3]
    at = lambda j, cam: next((x, y) for c, x, y in scene.obs[j] if c == cam)
    ghost = [_obs_line(77770 + k, *at(j, 0)) for k, j in enumerate(js)]
    extra = ["ghost_a"] + ghost + ["ghost_b"] + ghost + ["img1"] + [_obs_line(77770 + k, *at(j, 1)) for k, j in enumerate(js)]
    tp.write_text(tp.read_text() + "\n".join(extra) + "\n")
    cams = _check_pix4d(scene, tmp_path)
    assert 1 in [c["id"] for c in cams]


def test_pix4d_repeated_observation_stays_in_the_list(scene, tmp_path):
    scene.write_pix4d(tmp_path)
    tp = tmp_path / "proj_tp_pix4d.txt"
    lines = tp.read_text().split("\n")
    i1 = lines.index("img1")
    tp.write_text("\n".join(lines[:i1 + 2] + [lines[i1 + 1]] * 2 + lines[i1 + 2:]))
    cams = _check_pix4d(scene, tmp_path)
    w = next(c for c in cams if c["id"] == 1)["worldpoints"].tolist()
    assert w[0] == w[1] == w[2]


def test_pix4d_camera_with_two_valid_points_is_dropped(scene, tmp_path):
    """img2 keeps three observations, one of a point nobody else sees (not triangulated): two valid points, so no camera 2; a line
    whose id is shorter than two characters ends the file and ids starting with '-' are skipped"""
    scene.write_pix4d(tmp_path)
    tp = tmp_path / "proj_tp_pix4d.txt"
    lines = tp.read_text().split("\n")
    i2, i3 = lines.index("img2"), lines.index("img3")
    i6 = lines.index("img6")
    tp.write_text("\n".join(lines[:i2 + 3] + ["88000 10.5 20.5 1"] + lines[i3:i6] + ["-5 1 2 3", "x 1 2 3"] + lines[i6:]))
    cams = _check_pix4d(scene, tmp_path)
    ids = [c["id"] for c in cams]
    assert 2 not in ids and 6 not in ids and 7 not in ids and 1 in ids


# ---------------------------------------------------------------------------------------------- reader -> pipeline
def _run(scene, cams, neighbors_by_wps, const_depth=-1.0):
    L = line3d.Line3D(neighbors_by_worldpoints=neighbors_by_wps, use_gpu=True, device=0)
    try:
        for c in cams:
            L.add_image(c["id"], scene.width, scene.height, c["K"], c["R"], c["t"], c["median_depth"], c["list"], scene.synth.segs[c["view"]])
        L.match_images(const_reg_depth=const_depth)
        L.reconstruct_3d_lines(3, False)
        return L.lines()
    finally:
        L.close()


def _same_lines(a, b):
    assert len(a["lines"]) > 20
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def test_mavmap_pipeline(scene, tmp_path):
    scene.write_mavmap(tmp_path / "m.txt")
    read = line3d.read_mavmap(tmp_path / "m.txt")
    nb = lambda i: line3d.sequential_neighbors(i, scene.V, 4)
    a = _run(scene, [dict(c, view=i, median_depth=4.0, list=nb(i)) for i, c in enumerate(read)], False, 4.0)
    own = [dict(id=i, view=i, K=scene.K[i], R=scene.R_mav[i], t=scene.t_mav[i], median_depth=4.0, list=nb(i)) for i in range(scene.V)]
    _same_lines(a, _run(scene, own, False, 4.0))


def test_openmvg_pipeline(scene, tmp_path):
    (tmp_path / "o.json").write_text(scene.openmvg_text())
    read = line3d.read_openmvg(tmp_path / "o.json")
    a = _run(scene, [dict(c, view=c["id"] - 100, list=c["worldpoints"]) for c in read], True)
    Kf = lambda i: np.array([[scene.K[i][0, 0], 0, scene.K[i][0, 2]], [0, scene.K[i][0, 0], scene.K[i][1, 2]], [0, 0, 1]])
    own = [dict(id=c["id"], view=c["id"] - 100, K=Kf(c["id"] - 100), R=scene.R[c["id"] - 100], t=scene.t[c["id"] - 100], median_depth=c["median_depth"],
                list=c["worldpoints"]) for c in read]
    _same_lines(a, _run(scene, own, True))


def test_pix4d_pipeline(scene, tmp_path):
    scene.write_pix4d(tmp_path)
    read = line3d.read_pix4d(tmp_path, "proj")
    a = _run(scene, [dict(c, view=c["id"], list=c["worldpoints"]) for c in read], True)
    own = [dict(id=c["id"], view=c["id"], K=scene.K[c["id"]], R=scene.R[c["id"]], t=scene.t[c["id"]], median_depth=c["median_depth"], list=c["worldpoints"])
           for c in read]
    _same_lines(a, _run(scene, own, True))


def test_undistortion_with_the_readers_coefficients(ctx, scene, tmp_path):
    scene.write_pix4d(tmp_path)
    (tmp_path / "o.json").write_text(scene.openmvg_text())
    img = np.random.default_rng(2).integers(0, 256, (480, 640), dtype=np.uint8)
    for c in line3d.read_pix4d(tmp_path, "proj"):
        i = c["id"]
        a = ctx.undistort([img], c["K"], c["radial"], c["tangential"])[0]
        assert np.array_equal(a, ctx.undistort([img], scene.K[i], scene.radial[i], scene.tangential[i])[0])
    for c in line3d.read_openmvg(tmp_path / "o.json"):
        i = c["id"] - 100
        r, t = scene.openmvg_distortion(i)
        a = ctx.undistort([img], c["K"], c["radial"], c["tangential"])[0]
        assert np.array_equal(a, ctx.undistort([img], c["K"], r, t)[0])
