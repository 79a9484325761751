"""A synthetic SfM scene written out as a mavmap result file, an OpenMVG sfm_data.json and a Pix4D project (tests of the readers in
include/line3d_io.h), plus numpy restatements of what the reference's frontends compute from those files.

Every number that goes into a file is a dyadic rational written as its exact decimal expansion, so any correct parser (and
rapidjson's default, not full-precision, one) reads back the same double.  The cameras are those of line3dpp_b200.synth.make_scene, so
its 2D segments fit them.
"""
from __future__ import annotations

import json
import math
import os
from decimal import Decimal

import numpy as np

from line3dpp_b200 import synth


def q(v, bits):
    """v rounded to a multiple of 2^-bits"""
    return np.round(np.asarray(v, np.float64) * 2.0 ** bits) / 2.0 ** bits


def num(v) -> str:
    """the exact decimal expansion of a double"""
    s = format(Decimal(float(v)), "f")
    return s.rstrip("0").rstrip(".") if "." in s else s


def mul3(a, b):
    """3x3 product with the inner dimension summed left to right in IEEE double (the readers' order)"""
    return [[(a[r][0] * b[0][c] + a[r][1] * b[1][c]) + a[r][2] * b[2][c] for c in range(3)] for r in range(3)]


def neg_Rx(R, x):
    """-(R x), row sums left to right"""
    return np.array([-((R[r][0] * x[0] + R[r][1] * x[1]) + R[r][2] * x[2]) for r in range(3)])


def rotation_from_rpy(roll, pitch, yaw):
    """Line3D::rotationFromRPY: Rz * Ry * Rx of Eigen's AngleAxisd(angle, e_k).toRotationMatrix()"""
    def axis(a, k):
        s, c = math.sin(a), math.cos(a)
        R = [[0.0] * 3 for _ in range(3)]
        i, j = (k + 1) % 3, (k + 2) % 3
        R[k][k] = (1.0 - c) + c
        R[i][i] = c; R[j][j] = c; R[i][j] = -s; R[j][i] = s
        return R
    return np.array(mul3(mul3(axis(yaw, 2), axis(pitch, 1)), axis(roll, 0)))


def rpy_of(Rm):
    """roll, pitch, yaw with Rm = Rz(yaw) Ry(pitch) Rx(roll)"""
    return math.atan2(Rm[2, 1], Rm[2, 2]), -math.asin(max(-1.0, min(1.0, Rm[2, 0]))), math.atan2(Rm[1, 0], Rm[0, 0])


def decompose_restated(P):
    """line3D.cc:2784-2852 in numpy, step by step"""
    K = P[:, :3].copy()
    h = np.sqrt(K[2, 1] ** 2 + K[2, 2] ** 2); s, c = K[2, 1] / h, -K[2, 2] / h
    Rx = np.array([[1, 0, 0], [0, c, -s], [0, s, c]]); K = K @ Rx
    h = np.sqrt(K[2, 0] ** 2 + K[2, 2] ** 2); s, c = K[2, 0] / h, -K[2, 2] / h
    Ry = np.array([[c, 0, -s], [0, 1, 0], [s, 0, c]]); K = K @ Ry
    h = np.sqrt(K[1, 0] ** 2 + K[1, 1] ** 2); s, c = K[1, 0] / h, -K[1, 1] / h
    Rz = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]]); K = K @ Rz
    S = np.diag([-1.0 if K[i, i] < 0 else 1.0 for i in range(3)])
    K = K @ S
    R = (Rx @ Ry @ Rz @ S).T
    t = np.linalg.inv(K) @ P[:, 3]
    return K / K[2, 2], R, t


class Scene:
    """V cameras of synth.make_scene(V, N, seed, neighbors) with quantised intrinsics, rotations and centres, per-camera distortion and
    NP world points in [-1, 1]^3 (quantised), each observed by the cameras it projects into"""

    def __init__(self, V=8, N=150, seed=11, NP=240, neighbors="ring2"):
        self.synth = synth.make_scene(V, N, seed, neighbors)
        rng = np.random.default_rng(seed)
        self.V = V
        self.width, self.height = synth.WIDTH, synth.HEIGHT
        self.K = np.array([[[q(synth.FOCAL + 3.25 * i, 10), 0, q(synth.WIDTH / 2 + 0.5 * i, 10)], [0, q(synth.FOCAL - 1.5 * i, 10), q(synth.HEIGHT / 2 - 0.75 * i, 10)],
                            [0, 0, 1.0]] for i in range(V)])
        # mavmap stores the camera-to-world rotation as roll / pitch / yaw: its world-to-camera R_mav is the transpose of
        # rotationFromRPY.  OpenMVG and Pix4D store R itself, here quantised so that every decimal has at most 15 significant digits.
        self.rpy = [tuple(float(q(a, 30)) for a in rpy_of(self.synth.R[i].T)) for i in range(V)]
        self.C = q(np.einsum("vji,vj->vi", self.synth.R, -self.synth.t), 10)
        self.R_mav = np.array([rotation_from_rpy(*self.rpy[i]).T for i in range(V)])
        self.t_mav = np.array([neg_Rx(self.R_mav[i], self.C[i]) for i in range(V)])
        self.R = q(self.synth.R, 14)
        self.t = np.array([neg_Rx(self.R[i], self.C[i]) for i in range(V)])
        self.radial = q(rng.uniform(-0.05, 0.05, (V, 3)), 16)
        self.tangential = q(rng.uniform(-0.002, 0.002, (V, 2)), 18)
        self.X = q(rng.uniform(-1, 1, (NP, 3)), 10)
        self.obs = [[] for _ in range(NP)]                  # per point: (camera, x, y)
        for i in range(V):
            Xc = (self.R[i] @ self.X.T).T + self.t[i]
            u = (self.K[i] @ Xc.T).T
            xy = u[:, :2] / u[:, 2:]
            for j in np.flatnonzero((Xc[:, 2] > 0.1) & (xy[:, 0] >= 0) & (xy[:, 0] < self.width) & (xy[:, 1] >= 0) & (xy[:, 1] < self.height)):
                self.obs[j].append((i, float(q(xy[j, 0], 10)), float(q(xy[j, 1], 10))))

    # ---- mavmap
    def write_mavmap(self, path, comments=("# mavmap result", "# image, roll, pitch, ..."), tail=""):
        lines = list(comments)
        for i in range(self.V):
            f = [f"img{i}"] + [num(a) for a in self.rpy[i]] + ["47.1", "8.5", "400.25", "0"] + [num(c) for c in self.C[i]] + \
                ["1", "PINHOLE"] + [num(self.K[i][0, 0]), num(self.K[i][1, 1]), num(self.K[i][0, 2]), num(self.K[i][1, 2])]
            lines.append(" ".join(x + "," for x in f))
        open(path, "w").write("\n".join(lines) + "\n" + tail)

    # ---- OpenMVG
    MODELS = ("pinhole_radial_k3", "pinhole_radial_k1", "pinhole_brown_t2", "pinhole", "fisheye", None)

    def openmvg_distortion(self, i):
        """(radial, tangential) the reader must return for camera i (intrinsic i, model MODELS[i % 6]; None inherits the model before)"""
        m = self.MODELS[i % 6]
        if m is None:
            m = self.MODELS[(i - 1) % 6]
        r, t = np.zeros(3), np.zeros(2)
        if m == "pinhole_radial_k3": r = self.radial[i].copy()
        elif m == "pinhole_radial_k1": r[0] = self.radial[i][0]
        elif m == "pinhole_brown_t2": r, t = self.radial[i].copy(), self.tangential[i].copy()
        return r, t

    def openmvg_doc(self):
        D = float
        views, intr, extr, struct = [], [], [], []
        for i in range(self.V):
            views.append({"key": i, "value": {"polymorphic_id": 1073741824, "ptr_wrapper": {"id": 2147483649 + i, "data": {
                "local_path": "", "filename": f"img{i}.jpg", "width": self.width, "height": self.height, "id_view": 100 + i, "id_intrinsic": 10 + i,
                "id_pose": 50 + i}}}})
            m = self.MODELS[i % 6]
            data = {"width": self.width, "height": self.height, "focal_length": D(self.K[i][0, 0]), "principal_point": [D(self.K[i][0, 2]), D(self.K[i][1, 2])]}
            data["disto_k3"] = [D(v) for v in self.radial[i]]
            data["disto_k1"] = [D(self.radial[i][0])]
            data["disto_t2"] = [D(v) for v in self.radial[i]] + [D(v) for v in self.tangential[i]]
            val = {"polymorphic_id": 2147483649, "ptr_wrapper": {"id": 2147483700 + i, "data": data}}
            if m is not None:
                val["polymorphic_name"] = m
            intr.append({"key": 10 + i, "value": val})
            extr.append({"key": 50 + i, "value": {"rotation": [[D(v) for v in row] for row in self.R[i]], "center": [D(v) for v in self.C[i]]}})
        for j in range(len(self.X)):
            struct.append({"key": 7 * j + 3, "value": {"X": [D(v) for v in self.X[j]],
                                                      "observations": [{"key": 100 + c, "value": {"id_feat": j, "x": [D(x), D(y)]}} for c, x, y in self.obs[j]]}})
        return {"sfm_data_version": "0.3", "root_path": "/images", "views": views, "intrinsics": intr, "extrinsics": extr, "structure": struct,
                "control_points": []}

    def openmvg_text(self):
        """the document with every float as its exact decimal expansion"""
        def dump(o, ind):
            pad = "\n" + " " * ind
            if isinstance(o, dict):
                return "{" + ",".join(pad + " " + json.dumps(k) + ": " + dump(v, ind + 1) for k, v in o.items()) + pad + "}" if o else "{}"
            if isinstance(o, list):
                return "[" + ", ".join(dump(v, ind + 1) for v in o) + "]"
            if isinstance(o, float):
                return num(o)
            return json.dumps(o)
        text = dump(self.openmvg_doc(), 0)
        assert json.loads(text) == self.openmvg_doc()
        return text

    def openmvg_expected(self):
        """per camera (view order): wps (point keys) and the float median depth, as main_openmvg.cpp:326-398 computes them"""
        out = []
        for i in range(self.V):
            ids, d = [], []
            for j in range(len(self.X)):
                if any(c == i for c, _, _ in self.obs[j]):
                    ids.append(7 * j + 3)
                    dx, dy, dz = self.C[i] - self.X[j]
                    d.append(np.float32(math.sqrt(dx * dx + dy * dy + dz * dz)))
            d = np.sort(np.array(d, np.float32))
            out.append((ids, d[len(d) // 2] if len(d) else None))
        return out

    # ---- Pix4D
    def write_pix4d(self, folder, prefix="proj", noise=None, extra_tp=""):
        """<folder>/<prefix>_calibrated_camera_parameters.txt and _tp_pix4d.txt; point j has id str(1000 + j)"""
        os.makedirs(folder, exist_ok=True)
        L = ["Pix4D camera calibration file", "# description of the blocks", ""]
        for i in range(self.V):
            L.append(f"img{i}.JPG {self.width} {self.height}")
            L += [" ".join(num(v) for v in self.K[i][r]) for r in range(3)]
            L.append(" ".join(num(v) for v in self.radial[i]))
            L.append(" ".join(num(v) for v in self.tangential[i]))
            L.append(" ".join(num(v) for v in self.C[i]))
            L += [" ".join(num(v) for v in self.R[i][r]) for r in range(3)]
        open(os.path.join(folder, f"{prefix}_calibrated_camera_parameters.txt"), "w").write("\n".join(L) + "\n")
        T = []
        for i in range(self.V):
            T.append(f"img{i}")
            for j in range(len(self.X)):
                for c, x, y in self.obs[j]:
                    if c == i:
                        T.append(f"{1000 + j} {num(x)} {num(y)} 2.5")
        open(os.path.join(folder, f"{prefix}_tp_pix4d.txt"), "w").write("\n".join(T) + "\n" + extra_tp)


def pix4d_P(K, R, C):
    """P = K [R | -R C] of main_pix4d.cpp:266-272"""
    t = neg_Rx(R, C)
    return K @ np.hstack([R, t[:, None]])


def triangulate_restated(obs, P):
    """linearHomTriangulation for every point in numpy (eigh of the same A^T A): X [n, 3], valid [n]"""
    X = np.zeros((len(obs), 3)); valid = np.zeros(len(obs), np.int32)
    for j, o in enumerate(obs):
        if len(o) < 3:
            continue
        A = np.zeros((4, 4))
        for c, x, y in o:
            M = P[c]
            r1 = -M[1] + y * M[2]; r2 = M[0] - x * M[2]
            A += np.outer(r1, r1) + np.outer(r2, r2)
        v = np.linalg.eigh(A)[1][:, 0]
        X[j] = v[:3] / v[3]
        n = math.sqrt(X[j][0] ** 2 + X[j][1] ** 2 + X[j][2] ** 2)
        valid[j] = 1 if n > 1e-12 else 0
    return X, valid
