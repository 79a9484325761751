"""ctypes bindings of the CPU oracle (oracle/liboracle.so) and of the verbatim reference build (oracle/_ref/*.so).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs.  The product package (line3dpp_b200) never imports this module.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

MATCH_DT = np.dtype([("src_cam", "<u4"), ("src_seg", "<u4"), ("tgt_cam", "<u4"), ("tgt_seg", "<u4"),
                     ("overlap", "<f4"), ("score3D", "<f4"), ("d_p1", "<f4"), ("d_p2", "<f4"),
                     ("d_q1", "<f4"), ("d_q2", "<f4")])
SEG3D_DT = np.dtype([("line", "<i4"), ("_pad", "<i4"), ("p1", "<f8", 3), ("p2", "<f8", 3)])
RESID_DT = np.dtype([("line", "<i4"), ("cam", "<u4"), ("seg", "<u4")])


def build(ref: bool = True) -> None:
    """make -f oracle/Makefile (oracle always; _ref only when /root/reference is present)."""
    subprocess.check_call(["make", "-s", "-f", os.path.join(HERE, "Makefile"), "oracle"] + (["ref"] if ref else []))


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


_lib = None


def lib():
    global _lib
    if _lib is None:
        path = os.path.join(HERE, "liboracle.so")
        if not os.path.exists(path):
            build(ref=False)
        L = C.CDLL(path)
        L.orc_create.restype = C.c_void_p
        L.orc_match_lines_f32.restype = C.c_longlong
        L.orc_match_lines_f64.restype = C.c_longlong
        for n in ("orc_pair_evals", "orc_get_matches", "orc_get_scored", "orc_get_estimates", "orc_get_affinity",
                  "orc_get_affinity_raw", "orc_get_segments3d", "orc_get_residuals", "orc_get_collinear"):
            getattr(L, n).restype = C.c_longlong
        _lib = L
    return _lib


def ref_lib(variant: str = "nofma"):
    """The verbatim reference (cudawrapper.cu + sparsematrix.cc + clustering.cc) built by oracle/Makefile."""
    path = os.path.join(HERE, "_ref", f"libl3dref_{variant}.so")
    if not os.path.exists(path):
        return None
    L = C.CDLL(path)
    L.ref_match_lines.restype = C.c_longlong
    return L


def set_threads(n: int) -> None:
    lib().orc_set_threads(int(n))


# ------------------------------------------------------------------------------------------- kernel-level wrappers
def match_dense(fn, ls, lt, F, Rs, Rt, Cs, Ct, epi):
    """fn = lib().orc_match_dense_f32 or ref_lib().ref_match_dense.  Returns (depths[Ns,Nt,4], overlaps[Ns,Nt], ms)."""
    ls, lt = _f32(ls), _f32(lt)
    Ns, Nt = len(ls), len(lt)
    dep = np.empty((Ns, Nt, 4), np.float32)
    ov = np.empty((Ns, Nt), np.float32)
    ms = C.c_float(0)
    rc = fn(_p(ls), Ns, _p(lt), Nt, _p(_f32(F)), _p(_f32(Rs)), _p(_f32(Rt)), _p(_f32(Cs)), _p(_f32(Ct)),
            C.c_float(epi), _p(dep), _p(ov), C.byref(ms))
    assert rc == 0, rc
    return dep, ov, ms.value


def match_lines(fn, ls, lt, F, Rs, Rt, Cs, Ct, src_cam, tgt_cam, epi, knn, f64=False, cap=None):
    """Returns (counts[Ns], matches[Ns,cap] structured, total, wall_ms)."""
    conv = _f64 if f64 else _f32
    ls, lt = _f32(ls), _f32(lt)
    Ns, Nt = len(ls), len(lt)
    cap = cap or (knn if knn > 0 else Nt)
    counts = np.zeros(Ns, np.int32)
    out = np.zeros((Ns, cap), MATCH_DT)
    ms = C.c_double(0)
    fn.restype = C.c_longlong
    total = fn(_p(ls), Ns, _p(lt), Nt, _p(conv(F)), _p(conv(Rs)), _p(conv(Rt)), _p(conv(Cs)), _p(conv(Ct)),
               C.c_uint(src_cam), C.c_uint(tgt_cam), C.c_float(epi), C.c_int(knn), _p(counts), _p(out), cap,
               C.byref(ms))
    return counts, out, int(total), ms.value


def score_matches(fn, lines, matches4, ranges, reg_tgt, RtKinv, Cc, two_sigA_sqr, k, min_sim=0.5):
    lines, matches4, reg_tgt = _f32(lines), _f32(matches4), _f32(reg_tgt)
    ranges = np.ascontiguousarray(ranges, np.int32)
    M = len(matches4)
    scores = np.zeros(M, np.float32)
    ms = C.c_float(0)
    rc = fn(_p(lines), len(lines), _p(matches4), M, _p(ranges), _p(reg_tgt), _p(_f32(RtKinv)), _p(_f32(Cc)),
            C.c_float(two_sigA_sqr), C.c_float(k), C.c_float(min_sim), _p(scores), C.byref(ms))
    assert rc == 0, rc
    return scores, ms.value


def rdd(fn, ei, ej, ew, n, iters=None):
    """fn = lib().orc_rdd_f32 or ref_lib().ref_rdd (10 iterations).  iters (not None): lib().orc_rdd_f32_iters with that many
    iterations instead of fn.  Returns (out_i, out_j, out_w, wall_ms)."""
    ei, ej = np.ascontiguousarray(ei, np.int32), np.ascontiguousarray(ej, np.int32)
    ew = _f32(ew)
    ne = len(ei)
    oi, oj, ow = np.zeros(ne, np.int32), np.zeros(ne, np.int32), np.zeros(ne, np.float32)
    ms = C.c_double(0)
    if iters is None:
        rc = fn(ne, _p(ei), _p(ej), _p(ew), n, _p(oi), _p(oj), _p(ow), C.byref(ms))
    else:
        rc = lib().orc_rdd_f32_iters(ne, _p(ei), _p(ej), _p(ew), n, int(iters), _p(oi), _p(oj), _p(ow), C.byref(ms))
    assert rc == 0, rc
    return oi, oj, ow, ms.value


def collinear(fn, lines, dist_t):
    """fn = lib().orc_collinear_f32 / orc_collinear_f64 / ref_lib().ref_collinear.  Returns (C[N,N] uint8, ms)."""
    lines = _f32(lines)
    N = len(lines)
    Cm = np.zeros((N, N), np.uint8)
    ms = C.c_float(0)
    rc = fn(_p(lines), N, C.c_float(dist_t), _p(Cm), C.byref(ms))
    assert rc == 0, rc
    return Cm, ms.value


def cluster(fn, ei, ej, ew, n, c=3.0):
    ei, ej = np.ascontiguousarray(ei, np.int32), np.ascontiguousarray(ej, np.int32)
    lab = np.zeros(n, np.int32)
    rc = fn(len(ei), _p(ei), _p(ej), _p(_f32(ew)), n, C.c_float(c), _p(lab))
    assert rc == 0, rc
    return lab


# ------------------------------------------------------------------------------------------- pipeline wrapper
_MATCH_SOURCE_T = C.CFUNCTYPE(C.c_longlong, C.c_uint32, C.c_uint32, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int)

class OraclePipeline:
    """Restatement of L3DPP::Line3D (addImage / matchImages / reconstruct3Dlines) on explicit segments."""

    def __init__(self, neighbors_by_worldpoints=False, use_gpu=True, backend=None, match_source=None):
        """match_source: fn(src_cam, tgt_cam, Ns, Nt, kNN, cap) -> (counts int32[Ns], matches MATCH_DT[Ns, cap]) in place of
        matching every view pair (orc_set_match_source); its rows must obey what the matcher guarantees"""
        self.L = lib()
        self.ctx = C.c_void_p(self.L.orc_create(int(neighbors_by_worldpoints), int(use_gpu)))
        if match_source is not None:
            def source(src, tgt, Ns, Nt, knn, counts, out, cap):
                try:
                    cnt, m = match_source(int(src), int(tgt), int(Ns), int(Nt), int(knn), int(cap))
                    cnt = np.ascontiguousarray(cnt, np.int32)
                    m = np.ascontiguousarray(m, MATCH_DT)
                    assert cnt.shape == (Ns,) and m.shape == (Ns, cap) and (cnt >= 0).all() and (cnt <= cap).all()
                    C.memmove(counts, cnt.ctypes.data, cnt.nbytes)
                    C.memmove(out, m.ctypes.data, m.nbytes)
                    return int(cnt.sum())
                except Exception as e:  # noqa: BLE001 - must not unwind through the C frame; raised again by match_images
                    self._source_error = e
                    return 0
            self._source_error = None
            self._source = _MATCH_SOURCE_T(source)       # the library keeps the pointer: keep the callback alive
            self.L.orc_set_match_source(self.ctx, self._source)
        if backend is not None:   # verbatim reference kernels (oracle/_ref) instead of the CPU emulation
            g = lambda n: C.cast(getattr(backend, n), C.c_void_p)
            self.L.orc_set_backend(self.ctx, g("ref_match_lines"), g("ref_score_matches"), g("ref_rdd"))
            if hasattr(backend, "ref_collinear"):
                self.L.orc_set_collinear_backend(self.ctx, g("ref_collinear"))

    def __del__(self):
        if getattr(self, "ctx", None):
            self.L.orc_destroy(self.ctx)
            self.ctx = None

    def add_view(self, cam, width, height, K, R, t, median_depth, wps_or_neighbors, segs):
        lst = np.ascontiguousarray(wps_or_neighbors, np.uint32)
        segs = _f32(segs)
        return self.L.orc_add_view(self.ctx, C.c_uint(int(cam)), int(width), int(height), _p(_f64(K)), _p(_f64(R)),
                                   _p(_f64(t)), C.c_float(float(median_depth)), _p(lst), len(lst), _p(segs),
                                   len(segs))

    def add_scene(self, scene):
        for i in range(scene.num_views):
            rc = self.add_view(scene.cam_ids[i], scene.width, scene.height, scene.K[i], scene.R[i], scene.t[i],
                               scene.median_depth[i], scene.neighbors[i], scene.segs[i])
            assert rc == 0, rc

    def match_images(self, sigma_p=2.5, sigma_a=10.0, num_neighbors=10, epi_overlap=0.25, knn=10, const_reg_depth=-1.0):
        rc = self.L.orc_match_images(self.ctx, C.c_float(sigma_p), C.c_float(sigma_a), C.c_uint(num_neighbors),
                                     C.c_float(epi_overlap), C.c_int(knn), C.c_float(const_reg_depth))
        if getattr(self, "_source_error", None) is not None:
            raise self._source_error
        return rc

    def reconstruct(self, visibility_t=3, perform_diffusion=False, collinearity_t=-1.0, use_ceres=False, max_iter_ceres=250):
        return self.L.orc_reconstruct_opt(self.ctx, C.c_uint(visibility_t), int(perform_diffusion),
                                          C.c_float(collinearity_t), int(use_ceres), C.c_uint(max_iter_ceres))

    def opt_summary(self):
        s = np.zeros(8, np.float64)
        self.L.orc_get_opt_summary(self.ctx, _p(s))
        return s

    def pair_evals(self):
        return int(self.L.orc_pair_evals(self.ctx))

    def collinear(self, cam, nseg):
        """View::collin_ of a view as CSR (row_ptr[nseg+1], idx)"""
        row_ptr = np.zeros(nseg + 1, np.int64)
        n = self.L.orc_get_collinear(self.ctx, C.c_uint(int(cam)), _p(row_ptr), None, C.c_longlong(0))
        idx = np.zeros(max(int(n), 1), np.int32)
        if n > 0:
            self.L.orc_get_collinear(self.ctx, C.c_uint(int(cam)), _p(row_ptr), _p(idx), C.c_longlong(int(n)))
        return row_ptr, idx[:max(int(n), 0)]

    def pairs(self):
        n = self.L.orc_get_pairs(self.ctx, None, 0)
        a = np.zeros((n, 2), np.int32)
        self.L.orc_get_pairs(self.ctx, _p(a), n)
        return a

    def _matches(self, fn, cam):
        n = fn(self.ctx, C.c_uint(int(cam)), None, C.c_longlong(0))
        a = np.zeros(max(n, 0), MATCH_DT)
        if n > 0:
            fn(self.ctx, C.c_uint(int(cam)), _p(a), C.c_longlong(n))
        return a

    def matches(self, cam):
        return self._matches(self.L.orc_get_matches, cam)

    def scored(self, cam):
        return self._matches(self.L.orc_get_scored, cam)

    def view_info(self, cam):
        k, md = C.c_float(0), C.c_float(0)
        self.L.orc_get_view_info(self.ctx, C.c_uint(int(cam)), C.byref(k), C.byref(md))
        return k.value, md.value

    def estimates(self):
        n = self.L.orc_get_estimates(self.ctx, None, None, C.c_longlong(0))
        best = np.zeros(n, MATCH_DT)
        p = np.zeros((n, 6), np.float64)
        if n:
            self.L.orc_get_estimates(self.ctx, _p(best), _p(p), C.c_longlong(n))
        return best, p

    def _edges(self, fn):
        n = fn(self.ctx, None, None, None, C.c_longlong(0))
        ei, ej, ew = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.float32)
        if n:
            fn(self.ctx, _p(ei), _p(ej), _p(ew), C.c_longlong(n))
        return ei, ej, ew

    def affinity(self):
        return self._edges(self.L.orc_get_affinity)

    def affinity_raw(self):
        return self._edges(self.L.orc_get_affinity_raw)

    def local2global(self):
        n = self.L.orc_get_local2global(self.ctx, None, 0)
        a = np.zeros((n, 2), np.uint32)
        if n:
            self.L.orc_get_local2global(self.ctx, _p(a), n)
        return a

    def num_lines(self):
        return self.L.orc_num_lines(self.ctx)

    def segments3d(self):
        n = self.L.orc_get_segments3d(self.ctx, None, C.c_longlong(0))
        a = np.zeros(n, SEG3D_DT)
        if n:
            self.L.orc_get_segments3d(self.ctx, _p(a), C.c_longlong(n))
        return a

    def residuals(self):
        n = self.L.orc_get_residuals(self.ctx, None, C.c_longlong(0))
        a = np.zeros(n, RESID_DT)
        if n:
            self.L.orc_get_residuals(self.ctx, _p(a), C.c_longlong(n))
        return a

    def save_txt(self, path):
        return self.L.orc_save_txt(self.ctx, path.encode())


def optimize_lines(fn, p1p2, res_ptr, res_cam, res_xy, cams, max_iter=250, handle=None):
    """fn = lib().orc_optimize_lines (or the product's l3d_optimize_lines with handle = its context).
    Returns (p1p2_out[L,6], valid[L], summary[8])."""
    p1p2 = _f64(p1p2); res_xy = _f64(res_xy); cams = _f64(cams)
    res_ptr = np.ascontiguousarray(res_ptr, np.int64); res_cam = np.ascontiguousarray(res_cam, np.int32)
    L = len(p1p2)
    out = np.zeros((L, 6), np.float64); valid = np.zeros(L, np.int32); summ = np.zeros(8, np.float64)
    args = (L, _p(p1p2), _p(res_ptr), _p(res_cam), _p(res_xy), len(cams), _p(cams), int(max_iter), _p(out), _p(valid), _p(summ))
    rc = fn(*args) if handle is None else fn(handle, *args)
    assert rc == 0, rc
    return out, valid, summ


# ------------------------------------------------------------------------------------------- the reference's whole pipeline, verbatim
def ref_full_lib(variant: str = "cpu"):
    """oracle/_ref/libl3dref_full_{cpu,gpu}.so: /root/reference/line3D.cc + view.cc (+ the accelerator files) compiled verbatim
    against oracle/ref_shim (oracle/ref_full_harness.cu).  None if it has not been built."""
    path = os.path.join(HERE, "_ref", f"libl3dref_full_{variant}.so")
    if not os.path.exists(path):
        return None
    L = C.CDLL(path)
    L.rfl_create.restype = C.c_void_p
    for n in ("rfl_get_matches", "rfl_get_scored", "rfl_get_estimates", "rfl_get_affinity", "rfl_get_affinity_raw", "rfl_get_segments3d",
              "rfl_get_residuals", "rfl_get_collinear"):
        getattr(L, n).restype = C.c_longlong
    return L


class RefFullPipeline:
    """The UNMODIFIED L3DPP::Line3D (line3D.cc) behind the same dump interface as OraclePipeline.  variant "cpu": the
    reference's CPU code path (use_GPU is forced off by line3D.cc:49-53); "gpu": its CUDA code path (needs a GPU)."""

    def __init__(self, neighbors_by_worldpoints=False, use_gpu=False, variant="cpu", folder="/tmp/l3dref_full"):
        self.L = ref_full_lib(variant)
        if self.L is None:
            raise RuntimeError(f"oracle/_ref/libl3dref_full_{variant}.so not built")
        os.makedirs(folder, exist_ok=True)
        self.folder = folder
        self.ctx = C.c_void_p(self.L.rfl_create((folder.rstrip("/") + "/").encode(), int(neighbors_by_worldpoints), int(use_gpu)))

    def __del__(self):
        if getattr(self, "ctx", None):
            self.L.rfl_destroy(self.ctx)
            self.ctx = None

    def add_view(self, cam, width, height, K, R, t, median_depth, wps_or_neighbors, segs):
        lst = np.ascontiguousarray(wps_or_neighbors, np.uint32)
        segs = _f32(segs)
        return self.L.rfl_add_view(self.ctx, C.c_uint(int(cam)), int(width), int(height), _p(_f64(K)), _p(_f64(R)), _p(_f64(t)),
                                   C.c_float(float(median_depth)), _p(lst), len(lst), _p(segs), len(segs))

    def add_scene(self, scene):
        for i in range(scene.num_views):
            rc = self.add_view(scene.cam_ids[i], scene.width, scene.height, scene.K[i], scene.R[i], scene.t[i], scene.median_depth[i],
                               scene.neighbors[i], scene.segs[i])
            assert rc == 0, rc

    def match_images(self, sigma_p=2.5, sigma_a=10.0, num_neighbors=10, epi_overlap=0.25, knn=10, const_reg_depth=-1.0):
        return self.L.rfl_match_images(self.ctx, C.c_float(sigma_p), C.c_float(sigma_a), C.c_uint(num_neighbors), C.c_float(epi_overlap),
                                       C.c_int(knn), C.c_float(const_reg_depth))

    def reconstruct(self, visibility_t=3, perform_diffusion=False, collinearity_t=-1.0, use_ceres=False, max_iter_ceres=250):
        return self.L.rfl_reconstruct_opt(self.ctx, C.c_uint(visibility_t), int(perform_diffusion), C.c_float(collinearity_t), int(use_ceres),
                                          C.c_uint(max_iter_ceres))

    def pairs(self):
        n = self.L.rfl_get_pairs(self.ctx, None, 0)
        a = np.zeros((n, 2), np.int32)
        self.L.rfl_get_pairs(self.ctx, _p(a), n)
        return a

    def fundamental(self, src, tgt):
        F = np.zeros((3, 3))
        assert self.L.rfl_get_fundamental(self.ctx, C.c_uint(int(src)), C.c_uint(int(tgt)), _p(F)) == 0
        return F

    def neighbors(self, cam):
        a = np.zeros(4096, np.uint32)
        n = self.L.rfl_get_neighbors(self.ctx, C.c_uint(int(cam)), _p(a), len(a))
        return a[:n].copy()

    def _matches(self, fn, cam):
        n = fn(self.ctx, C.c_uint(int(cam)), None, C.c_longlong(0))
        a = np.zeros(max(n, 0), MATCH_DT)
        if n > 0:
            fn(self.ctx, C.c_uint(int(cam)), _p(a), C.c_longlong(n))
        return a

    def matches(self, cam):
        return self._matches(self.L.rfl_get_matches, cam)

    def scored(self, cam):
        return self._matches(self.L.rfl_get_scored, cam)

    def view_info(self, cam):
        k, md = C.c_float(0), C.c_float(0)
        self.L.rfl_get_view_info(self.ctx, C.c_uint(int(cam)), C.byref(k), C.byref(md))
        return k.value, md.value

    def view_geometry(self, cam):
        M, Cc = np.zeros((3, 3)), np.zeros(3)
        self.L.rfl_get_view_geometry(self.ctx, C.c_uint(int(cam)), _p(M), _p(Cc))
        return M, Cc

    def estimates(self):
        n = self.L.rfl_get_estimates(self.ctx, None, None, C.c_longlong(0))
        best, p = np.zeros(n, MATCH_DT), np.zeros((n, 6), np.float64)
        if n:
            self.L.rfl_get_estimates(self.ctx, _p(best), _p(p), C.c_longlong(n))
        return best, p

    def _edges(self, fn):
        n = fn(self.ctx, None, None, None, C.c_longlong(0))
        ei, ej, ew = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.float32)
        if n:
            fn(self.ctx, _p(ei), _p(ej), _p(ew), C.c_longlong(n))
        return ei, ej, ew

    def affinity(self):
        return self._edges(self.L.rfl_get_affinity)

    def affinity_raw(self):
        return self._edges(self.L.rfl_get_affinity_raw)

    def local2global(self):
        n = self.L.rfl_get_local2global(self.ctx, None, 0)
        a = np.zeros((n, 2), np.uint32)
        if n:
            self.L.rfl_get_local2global(self.ctx, _p(a), n)
        return a

    def clusters(self):
        n = self.L.rfl_get_clusters(self.ctx, None, None, None, 0)
        p, nr, rv = np.zeros((n, 6)), np.zeros(n, np.int32), np.zeros(n, np.uint32)
        if n:
            self.L.rfl_get_clusters(self.ctx, _p(p), _p(nr), _p(rv), n)
        return p, nr, rv

    def collinear(self, cam, nseg):
        row_ptr = np.zeros(nseg + 1, np.int64)
        n = self.L.rfl_get_collinear(self.ctx, C.c_uint(int(cam)), _p(row_ptr), None, C.c_longlong(0))
        idx = np.zeros(max(int(n), 1), np.int32)
        if n > 0:
            self.L.rfl_get_collinear(self.ctx, C.c_uint(int(cam)), _p(row_ptr), _p(idx), C.c_longlong(int(n)))
        return row_ptr, idx[:max(int(n), 0)]

    def num_lines(self):
        return self.L.rfl_num_lines(self.ctx)

    def segments3d(self):
        n = self.L.rfl_get_segments3d(self.ctx, None, C.c_longlong(0))
        a = np.zeros(n, SEG3D_DT)
        if n:
            self.L.rfl_get_segments3d(self.ctx, _p(a), C.c_longlong(n))
        return a

    def residuals(self):
        n = self.L.rfl_get_residuals(self.ctx, None, C.c_longlong(0))
        a = np.zeros(n, RESID_DT)
        if n:
            self.L.rfl_get_residuals(self.ctx, _p(a), C.c_longlong(n))
        return a

    def save(self, folder, txt=True, obj=False, stl=False):
        """the reference's own writers; returns createOutputFilename()"""
        buf = C.create_string_buffer(512)
        self.L.rfl_save(self.ctx, folder.encode(), int(txt), int(obj), int(stl), buf, 512)
        return buf.value.decode()
