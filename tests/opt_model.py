"""Float64 restatement of the line bundling (SURVEY.md §8f-4), written from the reference's optimization.h / optimization.cc and
Ceres' published trust-region defaults, independently of oracle/l3d_oracle.cc and csrc/l3d_optimize.cu.

  * Pluecker -> Cayley (optimization.cc:34-91) and Cayley -> end points (optimization.cc:213-298), vectorised over lines.
  * LineReprojectionError (optimization.h:66-158) vectorised over every residual block.  Derivatives come from complex-step
    differentiation, J[:, k] = Im r(x + i h e_k) / h with h = 1e-20: exact to rounding and a different derivation from the
    dual numbers of the library.  Every operation is analytic on complex input (sqrt(a*a + b*b), never hypot or abs), and
    every branch test compares the real part.
  * At |dot| >= 1 the dual-number acos has no finite derivative, so Ceres and the library take aw = 1 with a zero derivative
    (optimization.h:145).  Complex-step would differentiate straight through, so that rule is stated explicitly here.
  * HuberLoss(2) through Ceres' corrector (rho'' <= 0: residual and Jacobian scaled by sqrt(rho')), Jacobi scaling fixed at
    iteration zero, the Levenberg-Marquardt diagonal clamped to [1e-6, 1e32], one 4x4 Cholesky solve per line, and the
    trust-region controller with the library's rules: radius 1e4, min relative decrease 1e-3, function / gradient / parameter
    tolerance 1e-6 / 1e-10 / 1e-8, at most five consecutive invalid steps (each halves the radius and recomputes the diagonal),
    minimum radius 1e-32.

optimize() returns the library's 8-number summary, the end points and validity flags, and which rule stopped the run.
make_problem(kind, seed) builds fixed-seed problems that each reach one path of the bundling."""
import math

import numpy as np

EPS = 1e-12                       # L3D_EPS, and the omega / d conditions of optimization.h:91, 124
DBL_MAX = np.finfo(np.float64).max
DBL_MIN = np.finfo(np.float64).tiny
H_CS = 1e-20                      # complex-step size
KINDS = ("noisy", "outliers", "flipped", "parallel", "converged_zero", "converged_step", "mixed_free", "through_origin",
         "through_camera", "zero_length", "invalid")
SIZES = (1, 2, 127, 128, 129, 1023, 1024, 1025, 4097)


# ------------------------------------------------------------------------------------------------------------ conversions
def _normalized(v):
    """Eigen's normalize(): a zero vector stays zero"""
    n2 = (v * v).sum(-1, keepdims=True)
    return np.where(n2 > 0, v / np.sqrt(np.where(n2 > 0, n2, 1.0)), v)


def cayley_from_segments(p):
    """optimization.cc:34-91 for p [L, 6] -> (x [L, 4] = (omega, s), ok [L]).  ok = False: some coordinate is NaN, the line is
    kept constant at (-1, 0, 0, 0).  A line through the origin (|m| < EPS) takes the basis e1 = l x t, e2 = l x e1 with
    t = x (or y when |l_x| >= 0.9); the reference takes Eigen's FullPivLU kernel there, and omega = |m| < EPS makes every
    evaluation of such a line fail whichever basis is used."""
    P1, P2 = p[:, :3], p[:, 3:]
    l = _normalized(P2 - P1)
    m = np.cross(0.5 * (P1 + P2), l)
    mn = np.sqrt((m * m).sum(1))
    t = np.where((np.abs(l[:, 0]) < 0.9)[:, None], [1.0, 0.0, 0.0], [0.0, 1.0, 0.0])
    e1o = _normalized(np.cross(l, t))
    origin = (mn < EPS)[:, None]
    e1 = np.where(origin, e1o, _normalized(m))
    e2 = np.where(origin, np.cross(l, e1o), _normalized(np.cross(l, m)))
    Q = np.stack([l, e1, e2], 2)                                  # columns l, e1, e2
    I = np.eye(3)
    with np.errstate(all="ignore"):
        Bi = np.full_like(Q, np.nan)
        good = np.isfinite(Q).all((1, 2)) & (np.abs(np.linalg.det(np.where(np.isfinite(Q), Q, 0.0) + I)) > 0)
        if good.any():
            Bi[good] = np.linalg.inv(Q[good] + I)
        S = (Q - I) @ Bi
    x = np.stack([mn, S[:, 2, 1], S[:, 0, 2], S[:, 1, 0]], 1)
    ok = ~np.isnan(x).any(1)
    x[~ok] = (-1.0, 0.0, 0.0, 0.0)
    return x, ok


def segments_from_cayley(x, p_old):
    """optimization.cc:213-298 -> (p_out [L, 6], valid [L], axis [L]).  axis: 0 / 1 / 2 the dominant-axis case that placed the
    line, -1 the old end points were kept (omega < 0, omega ~ 0, or l ~ 0)."""
    L = len(x)
    P1, P2 = p_old[:, :3].copy(), p_old[:, 3:].copy()
    axis = np.full(L, -1)
    om, s = x[:, 0], x[:, 1:]
    nm = (s * s).sum(1)
    sk = np.zeros((L, 3, 3))
    sk[:, 0, 1], sk[:, 0, 2], sk[:, 1, 0], sk[:, 1, 2], sk[:, 2, 0], sk[:, 2, 1] = -s[:, 2], s[:, 1], s[:, 2], -s[:, 0], -s[:, 1], s[:, 0]
    with np.errstate(all="ignore"):
        Q = ((1.0 - nm)[:, None, None] * np.eye(3) + 2.0 * sk + 2.0 * s[:, :, None] * s[:, None, :]) / (1.0 + nm)[:, None, None]
        l, m = Q[:, :, 0], Q[:, :, 1] * om[:, None]
        a = np.abs(l)
        upd = ~(om < 0.0) & ~(np.abs(om) < EPS) & (a > EPS).any(1)
        Pm = 0.5 * (P1 + P2)
        cx = (a[:, 0] > a[:, 1]) & (a[:, 0] > a[:, 2])
        cy = ~cx & (a[:, 1] > a[:, 0]) & (a[:, 1] > a[:, 2])
        cz = ~cx & ~cy
        X = np.empty((L, 3))
        X[cx, 0] = Pm[cx, 0]
        X[cx, 2] = (-m[cx, 1] - X[cx, 0] * l[cx, 2]) / -l[cx, 0]
        X[cx, 1] = (m[cx, 2] - X[cx, 0] * l[cx, 1]) / -l[cx, 0]
        X[cy, 1] = Pm[cy, 1]
        X[cy, 2] = (m[cy, 0] - X[cy, 1] * l[cy, 2]) / -l[cy, 1]
        X[cy, 0] = (m[cy, 2] + X[cy, 1] * l[cy, 0]) / l[cy, 1]
        X[cz, 2] = Pm[cz, 2]
        X[cz, 1] = (m[cz, 0] + X[cz, 2] * l[cz, 1]) / l[cz, 2]
        X[cz, 0] = (-m[cz, 1] + X[cz, 2] * l[cz, 0]) / l[cz, 2]
    P1[upd], P2[upd] = X[upd] + l[upd], X[upd] - l[upd]
    axis[upd] = np.where(cx, 0, np.where(cy, 1, 2))[upd]
    d = P1 - P2
    valid = np.sqrt((d * d).sum(1)) > EPS
    return np.concatenate([P1, P2], 1), valid, axis


# ------------------------------------------------------------------------------------------------------------ residuals
def observations(xy):
    """optimization.cc:154-162: end points and the observed direction as a normal (-dir_y, dir_x); a zero direction stays zero"""
    d = _normalized(xy[:, 2:] - xy[:, :2])
    return np.stack([-d[:, 1], d[:, 0]], 1)


def residuals(x, cam, xy, nrm):
    """LineReprojectionError for B blocks: x [B, 4] (real or complex), cam [B, 16], xy [B, 4], nrm [B, 2] -> (r [B, 2], ok [B],
    branch [B]).  ok = False where the functor returns false (|omega| < EPS or d < EPS).  branch: 0 angle <= pi/2, 1 angle >
    pi/2 (folded to pi - angle), 2 |dot| >= 1 (aw = 1, constant)."""
    om, sx, sy, sz = x[:, 0], x[:, 1], x[:, 2], x[:, 3]
    R, C = cam[:, :9].reshape(-1, 3, 3), cam[:, 9:12]
    fx, fy, px, py = cam[:, 12], cam[:, 13], cam[:, 14], cam[:, 15]
    nm = sx * sx + sy * sy + sz * sz
    div = 1.0 / (1.0 + nm)
    l = [div * (1.0 - nm + 2.0 * sx * sx), div * (2.0 * sz + 2.0 * sy * sx), div * (-2.0 * sy + 2.0 * sz * sx)]
    m = [om * div * (-2.0 * sz + 2.0 * sx * sy), om * div * (1.0 - nm + 2.0 * sy * sy), om * div * (2.0 * sx + 2.0 * sz * sy)]
    mc = [m[0] - (C[:, 1] * l[2] - C[:, 2] * l[1]),                # m - C x l
          m[1] + (C[:, 0] * l[2] - C[:, 2] * l[0]),
          m[2] - (C[:, 0] * l[1] - C[:, 1] * l[0])]
    q = [R[:, i, 0] * mc[0] + R[:, i, 1] * mc[1] + R[:, i, 2] * mc[2] for i in range(3)]
    pl0, pl1 = fy * q[0], fx * q[1]
    pl2 = -fy * px * q[0] - fx * py * q[1] + fx * fy * q[2]
    with np.errstate(all="ignore"):
        d = np.sqrt(pl0 * pl0 + pl1 * pl1)
        ok = ~(np.abs(om.real) < EPS) & ~(d.real < EPS)
        dot = (pl0 * nrm[:, 0] + pl1 * nrm[:, 1]) / d
        finite = np.abs(dot.real) < 1.0
        dsafe = np.where(finite, dot, 0.0)
        ang = np.arccos(dsafe)
        flip = ang.real > math.pi / 2
        ang = np.where(flip, math.pi - ang, ang)
        aw = np.where(finite, np.exp(2.0 * ang), 1.0)
        r = np.stack([(pl0 * xy[:, 0] + pl1 * xy[:, 1] + pl2) / d * aw, (pl0 * xy[:, 2] + pl1 * xy[:, 3] + pl2) / d * aw], 1)
    branch = np.where(finite, np.where(flip, 1, 0), 2)
    return r, ok, branch


class _Problem:
    def __init__(self, p1p2, res_ptr, res_cam, res_xy, cams):
        self.p = np.asarray(p1p2, np.float64).reshape(-1, 6)
        self.ptr = np.asarray(res_ptr, np.int64)
        self.rc = np.asarray(res_cam, np.int64)
        self.xy = np.asarray(res_xy, np.float64).reshape(-1, 4)
        self.cams = np.asarray(cams, np.float64).reshape(-1, 16)
        self.L = len(self.p)


def _evaluate(P, free, x, jac, tally):
    """cost per line (0.5 sum rho), failed per line, and with jac the robustified gradient [L, 4] and J'J [L, 4, 4]"""
    L = P.L
    counts = np.diff(P.ptr)
    lines = np.repeat(np.arange(L), counts)
    blk = np.arange(P.ptr[-1])
    sel = free[lines]
    lob, blk = lines[sel], blk[sel]
    cam, xy = P.cams[P.rc[blk]], P.xy[blk]
    nrm = observations(xy)
    r, ok, branch = residuals(x[lob], cam, xy, nrm)
    failed = np.bincount(lob, ~ok, minlength=L) > 0
    r = np.where(ok[:, None], r, 0.0)
    with np.errstate(all="ignore"):
        s = r[:, 0] * r[:, 0] + r[:, 1] * r[:, 1]
        lin = s > 4.0
        sr = np.sqrt(s)
        rho = np.where(lin, 4.0 * sr - 4.0, s)
        rho1 = np.where(lin, np.fmax(DBL_MIN, 2.0 / sr), 1.0)
    cost = np.bincount(lob, 0.5 * rho, minlength=L)
    if tally is not None:
        tally["huber_quadratic"] += int((ok & ~lin).sum()); tally["huber_linear"] += int((ok & lin).sum())
        for b, name in enumerate(("angle_direct", "angle_flipped", "angle_nonfinite")):
            tally[name] += int((ok & (branch == b)).sum())
    if not jac:
        return cost, failed, None, None
    Jm = np.empty((len(blk), 2, 4))
    for k in range(4):
        xk = x[lob].astype(np.complex128)
        xk[:, k] += 1j * H_CS
        rk, _, _ = residuals(xk, cam, xy, nrm)
        Jm[:, :, k] = rk.imag / H_CS
    Jm[~ok] = 0.0
    with np.errstate(all="ignore"):
        w = np.sqrt(rho1)
        jr, rr = w[:, None, None] * Jm, w[:, None] * r
        gb = (jr * rr[:, :, None]).sum(1)
        Hb = np.einsum("bea,bec->bac", jr, jr)
    g = np.stack([np.bincount(lob, gb[:, k], minlength=L) for k in range(4)], 1)
    H = np.stack([np.bincount(lob, Hb[:, a, c], minlength=L) for a in range(4) for c in range(4)], 1).reshape(L, 4, 4)
    return cost, failed, g, H


def _cholesky_solve(A, b):
    """(A) y = b for a stack of symmetric 4x4 A by Cholesky; ok = False where a pivot is not > 0 or y is not finite"""
    n = len(A)
    Lc = np.zeros((n, 4, 4))
    ok = np.ones(n, bool)
    with np.errstate(all="ignore"):
        for i in range(4):
            for j in range(i + 1):
                s = A[:, i, j] - (Lc[:, i, :j] * Lc[:, j, :j]).sum(1)
                if i == j:
                    ok &= s > 0.0
                    Lc[:, i, i] = np.sqrt(np.where(s > 0.0, s, np.nan))
                else:
                    Lc[:, i, j] = s / Lc[:, j, j]
        z = np.zeros((n, 4)); y = np.zeros((n, 4))
        for i in range(4):
            z[:, i] = (b[:, i] - (Lc[:, i, :i] * z[:, :i]).sum(1)) / Lc[:, i, i]
        for i in range(3, -1, -1):
            y[:, i] = (z[:, i] - (Lc[:, i + 1:, i] * y[:, i + 1:]).sum(1)) / Lc[:, i, i]
    ok &= np.isfinite(y).all(1)
    return y, ok


def _fsum(v):
    return math.fsum(np.asarray(v, np.float64).ravel().tolist())


def optimize(p1p2, res_ptr, res_cam, res_xy, cams, max_iter=250):
    """LineOptimizer::optimize.  Returns a dict: summary (iterations, initial cost, final cost, termination 0 convergence /
    1 max_iter / 2 failure, accepted steps, free lines, final radius, 0), p1p2_out, valid, stop (the rule that ended the run),
    free, axis, branch tallies over every evaluation (tally) and at iteration zero (tally0), J'J at iteration zero (H0), steps
    (accepted / rejected / invalid) and the per-line costs at the start and the end (line_cost0, line_cost)."""
    P = _Problem(p1p2, res_ptr, res_cam, res_xy, cams)
    L = P.L
    x, ok = cayley_from_segments(P.p)
    free = ok & (np.diff(P.ptr) > 0)
    tally = dict(huber_quadratic=0, huber_linear=0, angle_direct=0, angle_flipped=0, angle_nonfinite=0)
    steps = dict(accepted=0, rejected=0, invalid=0)
    it = term = 0
    cost0 = cost = 0.0
    radius = 1e4
    line_cost0 = line_cost = np.zeros(L)
    H0, tally0 = None, None
    stop = "no free lines"
    if free.any() and max_iter >= 0:
        lc, failed, g, H = _evaluate(P, free, x, True, tally)
        tally0 = dict(tally)
        if failed.any():
            term, stop = 2, "initial evaluation failed"             # nothing is changed; no cost is reported
        else:
            line_cost0 = line_cost = lc
            cost0 = cost = _fsum(lc)
            H0 = H
            dH = np.einsum("lkk->lk", H)
            S = np.where(free[:, None], 1.0 / (1.0 + np.sqrt(dH)), 1.0)
            Ssq = S[:, :, None] * S[:, None, :]
            gmax = lambda g: float(np.fmax.reduce(np.abs(g[free]).ravel(), initial=0.0))  # noqa: E731  (NaN ignored, like fmax)
            decrease, reuse, invalid = 2.0, False, 0
            diag = np.zeros((L, 4))
            stop = "gradient tolerance" if gmax(g) <= 1e-10 else None
            while stop is None:
                if it >= max_iter:
                    term, stop = 1, "max_iter"
                    break
                if radius <= 1e-32:
                    stop = "minimum radius"
                    break
                it += 1
                with np.errstate(all="ignore"):
                    gs, Hs = (S * g)[free], (Ssq * H)[free]
                if not reuse:
                    diag[free] = np.fmin(np.fmax(np.einsum("lkk->lk", Hs), 1e-6), 1e32)
                reuse = True
                A = Hs + np.einsum("lk,kj->lkj", diag[free] / radius, np.eye(4))
                y, solved = _cholesky_solve(A, gs)
                d = -y
                with np.errstate(all="ignore"):
                    mc = -((d * gs).sum(1) + 0.5 * np.einsum("la,lab,lb->l", d, Hs, d))
                model_change = _fsum(mc[solved])
                if not solved.all() or not (model_change > 0.0):     # HandleInvalidStep
                    steps["invalid"] += 1
                    invalid += 1
                    if invalid >= 5:
                        term, stop = 2, "invalid steps"
                        break
                    radius *= 0.5
                    reuse = False
                    continue
                invalid = 0
                st = d * S[free]
                xc = x.copy()
                xc[free] = x[free] + st
                step_norm, x_norm = math.sqrt(_fsum(st * st)), math.sqrt(_fsum(x[free] * x[free]))
                lcc, cfail, _, _ = _evaluate(P, free, xc, False, tally)
                cand = DBL_MAX if cfail.any() else _fsum(lcc)
                if step_norm <= 1e-8 * (x_norm + 1e-8):
                    stop = "parameter tolerance"
                elif abs(cost - cand) <= 1e-6 * cost:
                    stop = "function tolerance"                      # the candidate is not applied
                if stop:
                    break
                quality = (cost - cand) / model_change
                if quality > 1e-3:                                   # HandleSuccessfulStep
                    steps["accepted"] += 1
                    x = xc
                    lc, failed, g, H = _evaluate(P, free, x, True, tally)
                    if failed.any():                                 # not reachable: the candidate was evaluated at this x
                        term, stop = 2, "evaluation failed"
                        break
                    line_cost, cost = lc, _fsum(lc)
                    radius = min(1e16, radius / max(1.0 / 3.0, 1.0 - (2.0 * quality - 1.0) ** 3))
                    decrease, reuse = 2.0, False
                    if gmax(g) <= 1e-10:
                        stop = "gradient tolerance"
                else:                                                # HandleUnsuccessfulStep
                    steps["rejected"] += 1
                    radius /= decrease
                    decrease *= 2.0
                    reuse = True
    p_out, valid, axis = segments_from_cayley(x, P.p)
    summary = np.array([it, cost0, cost, term, steps["accepted"], int(free.sum()), radius, 0.0])
    return dict(summary=summary, p1p2_out=p_out, valid=valid.astype(np.int32), stop=stop, free=free, axis=axis, tally=tally,
                tally0=tally0, H0=H0, steps=steps, line_cost0=line_cost0, line_cost=line_cost, x=x)


# ------------------------------------------------------------------------------------------------------------ problems
FOCAL, PX, PY = 800.0, 500.0, 400.0


def _camera(C, target, up):
    z = target - C; z = z / np.linalg.norm(z)
    xa = np.cross(up, z); xa = xa / np.linalg.norm(xa)
    ya = np.cross(z, xa)
    return np.concatenate([np.stack([xa, ya, z]).ravel(), C, [FOCAL, FOCAL, PX, PY]])


def _cameras(rng, n):
    out = []
    for _ in range(n):
        d = rng.normal(size=3); d /= np.linalg.norm(d)
        up = np.cross(d, rng.normal(size=3))
        out.append(_camera(d * rng.uniform(9.0, 12.0), rng.uniform(-0.5, 0.5, 3), up / np.linalg.norm(up)))
    return np.array(out)


def _project(cams, X):
    """pinhole projection of points X [B, 3] into cams [B, 16] (x_c = R (X - C))"""
    R, C = cams[:, :9].reshape(-1, 3, 3), cams[:, 9:12]
    q = np.einsum("bij,bj->bi", R, X - C)
    return np.stack([cams[:, 12] * q[:, 0] / q[:, 2] + cams[:, 14], cams[:, 13] * q[:, 1] / q[:, 2] + cams[:, 15]], 1)


def _scene(rng, counts, ncam=12, noise=1.0, perturb=0.02):
    """random 3D lines in [-2, 2]^3 seen by `ncam` cameras 9-12 units away; counts[i] observed sub-segments of line i with
    `noise` px of Gaussian noise; the start is the true segment with `perturb` units of noise on its end points"""
    counts = np.asarray(counts, np.int64)
    L = len(counts)
    cams = _cameras(rng, ncam)
    ctr = rng.uniform(-2.0, 2.0, (L, 3))
    dr = rng.normal(size=(L, 3)); dr /= np.linalg.norm(dr, axis=1, keepdims=True)
    half = rng.uniform(0.5, 1.5, L)[:, None]
    A, B = ctr - half * dr, ctr + half * dr
    lines = np.repeat(np.arange(L), counts)
    nr = len(lines)
    rc = rng.integers(0, ncam, nr)
    t1, t2 = rng.uniform(0.0, 0.4, nr)[:, None], rng.uniform(0.6, 1.0, nr)[:, None]
    a, b = A[lines] + t1 * (B - A)[lines], A[lines] + t2 * (B - A)[lines]
    xy = np.concatenate([_project(cams[rc], a), _project(cams[rc], b)], 1) + rng.normal(0.0, noise, (nr, 4))
    p = np.concatenate([A, B], 1) + rng.normal(0.0, perturb, (L, 6))
    ptr = np.concatenate([[0], np.cumsum(counts)])
    return dict(p1p2=p, res_ptr=ptr, res_cam=rc.astype(np.int32), res_xy=xy, cams=cams)


def _axis_scene(rng, n_lines, n_cams, shift):
    """lines along the x axis through (0, 0, Z), Z integer, seen by cameras with R = I at integer centres (cx, 0, cz): the Cayley
    coordinates are (Z, 0, 0, 0) exactly and every projection is a horizontal image line.  Each line is observed as horizontal
    segments, the exact projections of the same line moved to (0, dy, Z + dz) with (dy, dz) = shift(rng), so the projected and
    observed normals are parallel EXACTLY at the start (|dot| == 1, aw = 1); with shift 0 every residual is exactly 0."""
    cams = np.array([np.concatenate([np.eye(3).ravel(), [float(rng.integers(-3, 4)), 0.0, float(-rng.integers(8, 12))], [FOCAL, FOCAL, PX, PY]])
                     for _ in range(n_cams)])
    p, rc, xy, ptr = [], [], [], [0]
    for i in range(n_lines):
        Z = float(rng.integers(1, 4))
        dy, dz = shift(rng)
        p.append([-1.0, 0.0, Z, 1.0, 0.0, Z])
        for c in rng.choice(n_cams, 3 + i % 3, replace=False):
            y = PY + FOCAL * dy / (Z + dz - cams[c, 11])              # the projected line: y = py + fy (Y - cy) / (Z - cz)
            x1 = float(rng.integers(200, 400)); x2 = x1 + float(rng.integers(100, 300))
            rc.append(c); xy.append([x1, y, x2, y])
        ptr.append(len(rc))
    return dict(p1p2=np.array(p), res_ptr=np.array(ptr), res_cam=np.array(rc, np.int32), res_xy=np.array(xy), cams=cams)


def _add_axis_line(pr, i, C):
    """make line i of pr the x axis line through (0, 0, 3) (Cayley coordinates (3, 0, 0, 0) exactly) and its first residual an
    observation of it on the projected line y = py by a new camera with R = I at the integer centre C"""
    pr["p1p2"][i] = [-1.0, 0.0, 3.0, 1.0, 0.0, 3.0]
    pr["cams"] = np.concatenate([pr["cams"], [np.concatenate([np.eye(3).ravel(), C, [FOCAL, FOCAL, PX, PY]])]])
    r0 = pr["res_ptr"][i]
    pr["res_cam"][r0] = len(pr["cams"]) - 1
    pr["res_xy"][r0] = [300.0, PY, 600.0, PY]


def make_problem(kind, seed=0):
    """fixed-seed problem of one kind (KINDS, or "sizes_<L>" with L in SIZES); see the module doc and test_opt_model_cpu.py"""
    rng = np.random.default_rng(seed + 1000 * (KINDS.index(kind) if kind in KINDS else 99))
    if kind.startswith("sizes_"):
        return _scene(rng, rng.integers(3, 9, int(kind[6:])), noise=0.5)
    if kind == "noisy":                                  # ragged 1-200 residuals, one line with 1000
        counts = rng.integers(1, 201, 300); counts[17] = 1000
        return _scene(rng, counts)
    if kind == "outliers":                               # ~20 % of the blocks moved tens of px: both Huber branches
        pr = _scene(rng, rng.integers(2, 40, 120))
        out = rng.random(len(pr["res_xy"])) < 0.2
        pr["res_xy"][out] += rng.uniform(20.0, 60.0, (out.sum(), 1)) * rng.choice([-1.0, 1.0], (out.sum(), 4))
        return pr
    if kind == "flipped":                                # end points swapped on about half the observations: angle > pi/2
        pr = _scene(rng, rng.integers(2, 40, 120))
        sw = rng.random(len(pr["res_xy"])) < 0.5
        pr["res_xy"][sw] = pr["res_xy"][sw][:, [2, 3, 0, 1]]
        return pr
    if kind == "parallel":                               # |dot| == 1 at iteration zero, the observations off the start line
        return _axis_scene(rng, 12, 6, lambda r: tuple(r.uniform(-0.1, 0.1, 2)))
    if kind == "converged_zero":                         # every residual and the gradient exactly 0
        return _axis_scene(rng, 12, 6, lambda r: (0.0, 0.0))
    if kind == "converged_step":                         # observations 1e-8 px from the start line: the first step is tiny
        return _scene(rng, rng.integers(5, 30, 60), noise=1e-8, perturb=0.0)
    if kind == "mixed_free":
        pr = _scene(rng, rng.integers(1, 20, 80))        # lines 0 mod 7 get no residuals below
        counts = np.diff(pr["res_ptr"])
        keep = np.concatenate([np.full(c, i % 7 != 0) for i, c in enumerate(counts)])
        counts[::7] = 0
        pr["res_cam"], pr["res_xy"] = pr["res_cam"][keep], pr["res_xy"][keep]
        pr["res_ptr"] = np.concatenate([[0], np.cumsum(counts)])
        pr["p1p2"][3::7, 4] = np.nan                     # NaN Cayley coordinates: constant, end points kept
        pr["p1p2"][7::14, 3:] = pr["p1p2"][7::14, :3]    # P1 == P2 without residuals: not free, valid = 0
        return pr
    if kind == "through_origin":                         # mid point 0: m = 0, omega = 0, the first evaluation fails
        pr = _scene(rng, rng.integers(2, 20, 40))
        pr["p1p2"][11] = [-0.5, 0.25, -1.0, 0.5, -0.25, 1.0]
        return pr
    if kind == "through_camera":                         # line 9 runs through the centre of a camera that observes it: d == 0
        pr = _scene(rng, rng.integers(2, 20, 40))
        _add_axis_line(pr, 9, [1.0, 0.0, 3.0])
        return pr
    if kind == "zero_length":                            # P1 == P2 with residuals: l = 0, omega = 0, the first evaluation fails
        pr = _scene(rng, rng.integers(2, 20, 40))
        pr["p1p2"][6, 3:] = pr["p1p2"][6, :3]
        return pr
    if kind == "invalid":                                # r == 0 exactly but |J| ~ 1e160: J'J overflows, every solve fails
        pr = _scene(rng, rng.integers(2, 20, 40))
        _add_axis_line(pr, 4, [0.0, 0.0, -9.0])
        pr["res_xy"][pr["res_ptr"][4]] = [1e160, PY, 1e160 + 1e150, PY]
        return pr
    raise ValueError(kind)
