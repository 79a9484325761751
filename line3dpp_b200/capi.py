"""ctypes binding of libl3d_b200.so (include/l3d_capi.h, include/l3dpp_capi.h).  Thin: no arithmetic happens in Python.

The library is REQUIRED: importing this module builds it if the .so is missing and raises if that fails; creating a
context raises if there is no usable CUDA device.  There is no CPU fallback anywhere in this package.
Every function the two headers declare gets its argtypes / restype from its declaration when the library is loaded.
"""
from __future__ import annotations

import ctypes as C
import os
import re
import numpy as np

from . import build as _build

HERE = os.path.dirname(os.path.abspath(__file__))
HEADERS = [os.path.join(os.path.dirname(HERE), "include", h) for h in ("l3d_capi.h", "l3dpp_capi.h")]


class ViewDesc(C.Structure):
    _fields_ = [("cam_id", C.c_uint32), ("width", C.c_int32), ("height", C.c_int32), ("nseg", C.c_int32),
                ("RtKinv", C.c_float * 9), ("C", C.c_float * 3), ("RtKinv_d", C.c_double * 9), ("C_d", C.c_double * 3),
                ("k", C.c_float), ("median_depth", C.c_float)]


class UndistortDesc(C.Structure):
    """l3d_undistort_desc: one 8-bit image and its camera"""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("channels", C.c_int32), ("src_pitch", C.c_int64), ("dst_pitch", C.c_int64),
                ("src", C.c_void_p), ("dst", C.c_void_p), ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("radial", C.c_double * 3), ("tangential", C.c_double * 2), ("model", C.c_int32), ("rational", C.c_double * 3),
                ("fisheye", C.c_double * 4)]


LENS_RADTAN, LENS_FISHEYE = 0, 1     # l3d_undistort_desc::model


def make_undistort_desc(width, height, channels, K, radial=(0, 0, 0), tangential=(0, 0), src=0, src_pitch=None, dst=0, dst_pitch=None,
                        model=LENS_RADTAN, rational=(0, 0, 0), fisheye=(0, 0, 0, 0)):
    """K: 3x3 camera matrix (fx, fy, cx, cy are read, skew is ignored); src / dst: addresses; pitches in bytes (default packed);
    model: LENS_RADTAN (radial k1 k2 k3, tangential p1 p2, rational k4 k5 k6) or LENS_FISHEYE (fisheye k1..k4)"""
    K = np.asarray(K, np.float64).reshape(3, 3)
    row = int(width) * int(channels)
    d = UndistortDesc()
    d.width, d.height, d.channels = int(width), int(height), int(channels)
    d.src_pitch = row if src_pitch is None else int(src_pitch)
    d.dst_pitch = row if dst_pitch is None else int(dst_pitch)
    d.src, d.dst = int(src) or None, int(dst) or None
    d.fx, d.fy, d.cx, d.cy = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])
    d.radial[:] = [float(v) for v in radial]
    d.tangential[:] = [float(v) for v in tangential]
    d.model = int(model)
    d.rational[:] = [float(v) for v in rational]
    d.fisheye[:] = [float(v) for v in fisheye]
    return d


def lens_desc_args(lens):
    """the make_undistort_desc keywords of a lens dict {"model": 0 | 1, "k": k1..k6 (radtan) or k1..k4 (fisheye), "p": p1, p2}, the
    layout of L3DPP::LensDistortion"""
    k = [float(v) for v in lens.get("k", ())] + [0.0] * 6
    p = [float(v) for v in lens.get("p", ())] + [0.0] * 2
    if int(lens.get("model", LENS_RADTAN)) == LENS_FISHEYE:     # k5, k6, p1, p2 go where l3d_undistort_u8 rejects them if nonzero
        return dict(model=LENS_FISHEYE, fisheye=k[:4], radial=k[4:6] + [0.0], tangential=p[:2])
    return dict(model=int(lens.get("model", LENS_RADTAN)), radial=k[:3], tangential=p[:2], rational=k[3:6])


class ImagePrepDesc(C.Structure):
    """l3d_image_prep_desc: one 8-bit image, its max_img_width and the grey output"""
    _fields_ = [("width", C.c_int32), ("height", C.c_int32), ("channels", C.c_int32), ("max_img_width", C.c_int32),
                ("src_pitch", C.c_int64), ("dst_pitch", C.c_int64), ("src", C.c_void_p), ("dst", C.c_void_p),
                ("out_width", C.c_int32), ("out_height", C.c_int32)]


def image_prep_size(width, height, max_img_width):
    """(out_width, out_height, resized) of l3d_image_prep_size: the size of the image line detection sees"""
    w, h = C.c_int32(), C.c_int32()
    rc = lib().l3d_image_prep_size(int(width), int(height), int(max_img_width), C.byref(w), C.byref(h))
    if rc < 0:
        raise L3DError(f"l3d_image_prep_size({width}, {height}, {max_img_width}) failed ({rc})")
    return w.value, h.value, bool(rc)


def make_image_prep_desc(width, height, channels, max_img_width, src=0, src_pitch=None, dst=0, dst_pitch=None):
    """src / dst: addresses; pitches in bytes (default packed); the output size is l3d_image_prep_size's"""
    ow, oh, _ = image_prep_size(width, height, max_img_width)
    d = ImagePrepDesc()
    d.width, d.height, d.channels, d.max_img_width = int(width), int(height), int(channels), int(max_img_width)
    d.src_pitch = int(width) * int(channels) if src_pitch is None else int(src_pitch)
    d.dst_pitch = ow if dst_pitch is None else int(dst_pitch)
    d.src, d.dst = int(src) or None, int(dst) or None
    d.out_width, d.out_height = ow, oh
    return d


def _image_rows(a):
    """(array, row pitch in bytes) of a uint8 HxW / HxWx3 image whose pixels are packed within each row; other layouts are copied"""
    a = np.asarray(a)
    if a.dtype != np.uint8 or a.ndim not in (2, 3) or (a.ndim == 3 and a.shape[2] != 3):
        raise ValueError("expected a uint8 HxW or HxWx3 image")
    c = 1 if a.ndim == 2 else 3
    if a.strides[1] != c or (a.ndim == 3 and a.strides[2] != 1) or a.strides[0] < a.shape[1] * c:
        a = np.ascontiguousarray(a)
    return a, a.strides[0]


REC_DT = np.dtype([("tgt_seg", "<u4"), ("overlap", "<f4"), ("d_p1", "<f4"), ("d_p2", "<f4"), ("d_q1", "<f4"),
                   ("d_q2", "<f4")])
MATCH_DT = np.dtype([("src_cam", "<u4"), ("src_seg", "<u4"), ("tgt_cam", "<u4"), ("tgt_seg", "<u4"),
                     ("overlap", "<f4"), ("score3D", "<f4"), ("d_p1", "<f4"), ("d_p2", "<f4"),
                     ("d_q1", "<f4"), ("d_q2", "<f4")])

_lib = None


class L3DError(RuntimeError):
    pass


_VALUE_TYPES = {"int": C.c_int, "int32_t": C.c_int, "unsigned int": C.c_uint, "uint32_t": C.c_uint, "long long": C.c_longlong,
                "int64_t": C.c_longlong, "size_t": C.c_size_t, "float": C.c_float, "double": C.c_double}


def declarations(path):
    """{name: (restype, argtypes)} of the file-scope declarations `ret name(params);` of l3d_* / l3dpp_* functions in a C header.
    Every pointer (function-pointer typedefs of the header and `T* const*` included) is c_void_p, a `const char*` result c_char_p,
    the other types those of _VALUE_TYPES; any other spelling raises, naming the declaration."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", open(path).read(), flags=re.S)
    text = re.sub(r"^[ \t]*#.*$", " ", text, flags=re.M)
    text = re.sub(r'extern\s*"C"\s*\{|\}', " ", text)
    fn_ptrs, out = set(), {}

    def c_type(spelling, decl, result=False):
        t = " ".join(spelling.replace("*", " * ").split())
        if result and t in ("void", "const char *"):
            return None if t == "void" else C.c_char_p
        if "*" in t or t in fn_ptrs:
            return C.c_void_p
        if t not in _VALUE_TYPES:
            raise L3DError(f"{os.path.basename(path)}: no ctypes type for `{spelling}` in `{decl};`")
        return _VALUE_TYPES[t]

    for decl in (" ".join(s.split()) for s in text.split(";")):
        if decl.startswith("typedef"):
            fn_ptrs.update(re.findall(r"\(\s*\*\s*(\w+)\s*\)\s*\(", decl))
        elif re.search(r"\bl3d(pp)?_\w+\s*\(", decl):
            m = re.fullmatch(r"([\w ]+?\**) ?(l3d(?:pp)?_\w+) ?\(([^()]*)\)", decl)
            if m is None:
                raise L3DError(f"{os.path.basename(path)}: `{decl};` is not a declaration `ret name(params);`")
            params = [] if m.group(3).strip() == "void" else [p.replace("*", "* ").split() for p in m.group(3).split(",")]
            # a parameter's last word is its name, unless the words are a type on their own or end a pointer type
            types = [w if len(w) <= 1 or " ".join(w) in _VALUE_TYPES or w[-1].endswith("*") else w[:-1] for w in params]
            out[m.group(2)] = (c_type(m.group(1), decl, result=True), [c_type(" ".join(w), decl) for w in types])
    return out


def bind(L, headers=HEADERS):
    """L (a CDLL) with the argtypes / restype of every function the headers declare; raises if L lacks one"""
    for h in headers:
        for name, (restype, argtypes) in declarations(h).items():
            f = getattr(L, name)
            f.restype, f.argtypes = restype, argtypes
    return L


def lib():
    global _lib
    if _lib is None:
        _lib = bind(C.CDLL(os.environ.get("L3D_LIB") or _build.build()))     # L3D_LIB: load a tile-sweep variant instead
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def make_view_descs(cam_ids, widths, heights, nsegs, RtKinv_d, C_untranslated_d, C_work_d, k, median_depth):
    """Pack camera blocks (already computed by the host side, in double) into l3d_view_desc[]."""
    V = len(cam_ids)
    arr = (ViewDesc * V)()
    for v in range(V):
        d = arr[v]
        d.cam_id, d.width, d.height, d.nseg = int(cam_ids[v]), int(widths[v]), int(heights[v]), int(nsegs[v])
        R = np.asarray(RtKinv_d[v], np.float64).reshape(9)
        d.RtKinv[:] = R.astype(np.float32).tolist()
        d.RtKinv_d[:] = R.tolist()
        d.C[:] = np.asarray(C_untranslated_d[v], np.float64).astype(np.float32).tolist()
        d.C_d[:] = np.asarray(C_work_d[v], np.float64).tolist()
        d.k = float(k[v])
        d.median_depth = float(median_depth[v])
    return arr


class Context:
    """One l3d_ctx (one GPU)."""

    def __init__(self, device: int = 0):
        self.L = lib()
        h = C.c_void_p()
        rc = self.L.l3d_ctx_create(int(device), C.byref(h))
        if rc != 0 or not h:
            raise L3DError(f"l3d_ctx_create(device={device}) failed with {rc}: no usable CUDA device "
                           "(libl3d_b200 has no CPU fallback)")
        self.h = h
        self._keep = []

    def close(self):
        if getattr(self, "h", None):
            self.L.l3d_ctx_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _chk(self, rc, what):
        if rc < 0:
            raise L3DError(f"{what} failed ({rc}): {self.L.l3d_last_error(self.h).decode()}")
        return rc

    @property
    def stream(self) -> int:
        return int(self.L.l3d_stream(self.h) or 0)

    def sync(self):
        self._chk(self.L.l3d_sync(self.h), "l3d_sync")

    def launch_count(self) -> int:
        return int(self.L.l3d_launch_count(self.h))

    # ---- views
    def set_views(self, descs, segs_list):
        V = len(descs)
        segs = [np.ascontiguousarray(s, np.float32) for s in segs_list]
        ptrs = (C.c_void_p * V)(*[s.ctypes.data for s in segs])
        self._keep = [descs, segs]
        self._chk(self.L.l3d_set_views(self.h, V, descs, ptrs), "l3d_set_views")

    def set_views_flat(self, descs, segs_flat_ptr: int, on_device: bool):
        self._keep = [descs]
        self._chk(self.L.l3d_set_views_flat(self.h, len(descs), descs, segs_flat_ptr, int(on_device)),
                  "l3d_set_views_flat")

    def update_view_params(self, descs):
        self._chk(self.L.l3d_update_view_params(self.h, len(descs), descs), "l3d_update_view_params")

    # ---- matching
    def match_pairs(self, pairs, F, epi_overlap=0.25, knn=10):
        pairs = np.ascontiguousarray(pairs, np.int32).reshape(-1, 2)
        F = np.ascontiguousarray(F, np.float32).reshape(-1, 9)
        assert len(pairs) == len(F)
        self._chk(self.L.l3d_match_pairs(self.h, len(pairs), _p(pairs), _p(F), epi_overlap, int(knn)),
                  "l3d_match_pairs")
        self._knn = int(self.L.l3d_match_stride(self.h))

    def match_pairs_range(self, pairs, F, first, last, epi_overlap=0.25, knn=10):
        """sharded form: stage all pairs, evaluate only [first, last) here (include/l3d_capi.h)"""
        pairs = np.ascontiguousarray(pairs, np.int32).reshape(-1, 2)
        F = np.ascontiguousarray(F, np.float32).reshape(-1, 9)
        assert len(pairs) == len(F)
        self._chk(self.L.l3d_match_pairs_range(self.h, len(pairs), _p(pairs), _p(F), epi_overlap, int(knn), int(first), int(last)),
                  "l3d_match_pairs_range")
        self._knn = int(self.L.l3d_match_stride(self.h))

    def match_pairs_f64(self, pairs, Fd, epi_overlap=0.25, knn=10, first=0, last=None):
        """REF_CPU semantics: matchingCPU's double arithmetic (line3D.cc:900-1015) with double fundamental matrices"""
        pairs = np.ascontiguousarray(pairs, np.int32).reshape(-1, 2)
        Fd = np.ascontiguousarray(Fd, np.float64).reshape(-1, 9)
        assert len(pairs) == len(Fd)
        last = len(pairs) if last is None else last
        self._chk(self.L.l3d_match_pairs_f64(self.h, len(pairs), _p(pairs), _p(Fd), epi_overlap, int(knn), int(first), int(last)),
                  "l3d_match_pairs_f64")
        self._knn = int(self.L.l3d_match_stride(self.h))

    def match_pairs_host(self, pairs, F, counts_ptr: int, recs_ptr: int, epi_overlap=0.25, knn=10, chunks=8):
        """match + overlapped download into host memory at the given addresses (pinned for real overlap); asynchronous"""
        pairs = np.ascontiguousarray(pairs, np.int32).reshape(-1, 2)
        F = np.ascontiguousarray(F, np.float32).reshape(-1, 9)
        assert len(pairs) == len(F)
        self._chk(self.L.l3d_match_pairs_host(self.h, len(pairs), _p(pairs), _p(F), epi_overlap, int(knn), counts_ptr, recs_ptr, int(chunks)),
                  "l3d_match_pairs_host")
        self._knn = int(knn)

    def match_device_buffers(self):
        """(counts_ptr, recs_ptr) device addresses of the last match result"""
        a, b = C.c_void_p(), C.c_void_p()
        self._chk(self.L.l3d_match_device_buffers(self.h, C.byref(a), C.byref(b)), "l3d_match_device_buffers")
        return a.value or 0, b.value or 0

    def match_gather(self, sources, pair_bounds):
        """l3d_match_gather: bring the rows of `sources` (Contexts, this one allowed), source i having matched the pairs
        [pair_bounds[i], pair_bounds[i+1]) of this context's pair list, into this context; asynchronous on its stream"""
        b = np.ascontiguousarray(pair_bounds, np.int32)
        if len(b) != len(sources) + 1:
            raise ValueError("pair_bounds needs one entry per source + 1")
        hs = (C.c_void_p * len(sources))(*[s.h.value for s in sources])
        self._chk(self.L.l3d_match_gather(self.h, len(sources), hs, _p(b)), "l3d_match_gather")
        self._knn = int(self.L.l3d_match_stride(self.h))

    def match_restride(self, stride=0) -> int:
        """l3d_match_restride: re-lay the records at `stride` slots per row (<= 0: the longest row); returns the stride"""
        self._knn = int(self._chk(self.L.l3d_match_restride(self.h, int(stride)), "l3d_match_restride"))
        return self._knn

    def pair_row_offsets(self, num_pairs):
        out = np.zeros(num_pairs + 1, np.int64)
        self._chk(self.L.l3d_pair_row_offsets(self.h, _p(out)), "l3d_pair_row_offsets")
        return out

    def match_total_rows(self) -> int:
        return int(self.L.l3d_match_total_rows(self.h))

    def match_pair_evals(self) -> int:
        return int(self.L.l3d_match_pair_evals(self.h))

    def match_counts(self):
        out = np.zeros(max(self.match_total_rows(), 0), np.int32)
        total = self._chk(self.L.l3d_get_match_counts(self.h, _p(out)), "l3d_get_match_counts")
        return out, int(total)

    def pair_matches(self, pair: int, ns: int):
        counts = np.zeros(ns, np.int32)
        recs = np.zeros((ns, self._knn), REC_DT)
        self._chk(self.L.l3d_get_pair_matches(self.h, int(pair), _p(counts), _p(recs)), "l3d_get_pair_matches")
        return counts, recs

    def matches_csr(self, row_ptr=None, recs=None):
        rows = self.match_total_rows()
        if row_ptr is None:
            row_ptr = np.zeros(rows + 1, np.int64)
        cap = 0 if recs is None else len(recs)
        total = self._chk(self.L.l3d_get_matches_csr(self.h, _p(row_ptr), _p(recs), cap),
                          "l3d_get_matches_csr")
        if recs is None or total > cap:
            recs = np.zeros(total, REC_DT)
            total = self._chk(self.L.l3d_get_matches_csr(self.h, _p(row_ptr), _p(recs), len(recs)),
                              "l3d_get_matches_csr")
        return row_ptr, recs[:total]

    def matches_csr_raw(self, row_ptr_ptr: int, recs_ptr: int, capacity: int) -> int:
        return int(self._chk(self.L.l3d_get_matches_csr(self.h, row_ptr_ptr, recs_ptr, capacity), "l3d_get_matches_csr"))

    def rdd(self, n, ei, ej, ew, iters=10):
        """l3d_rdd: returns (out_i, out_j, out_w, device ms of the diffusion iterations)"""
        ei = np.ascontiguousarray(ei, np.int32); ej = np.ascontiguousarray(ej, np.int32); ew = np.ascontiguousarray(ew, np.float32)
        oi, oj, ow = np.empty_like(ei), np.empty_like(ej), np.empty_like(ew)
        ms = C.c_float(0)
        self._chk(self.L.l3d_rdd(self.h, int(n), len(ei), _p(ei), _p(ej), _p(ew), int(iters), _p(oi), _p(oj), _p(ow),
                                 C.byref(ms)), "l3d_rdd")
        return oi, oj, ow, ms.value

    def find_collinear(self, dist_t: float, semantics: int = 0):
        """l3d_find_collinear for all views (semantics 0 = REF_GPU float kernel, 1 = REF_CPU); dist_t <= 0 switches the links off"""
        self._chk(self.L.l3d_find_collinear(self.h, dist_t, int(semantics)), "l3d_find_collinear")
        return int(self.L.l3d_collinear_total(self.h))

    def collinear(self, view: int, nseg: int):
        """View::collin_ of one view as CSR (row_ptr[nseg+1], idx)"""
        row_ptr = np.zeros(nseg + 1, np.int64)
        n = self._chk(self.L.l3d_get_collinear(self.h, int(view), _p(row_ptr), None, 0), "l3d_get_collinear")
        idx = np.zeros(max(int(n), 1), np.int32)
        if n > 0:
            self._chk(self.L.l3d_get_collinear(self.h, int(view), _p(row_ptr), _p(idx), n), "l3d_get_collinear")
        return row_ptr, idx[:int(n)]

    def optimize_lines(self, p1p2, res_ptr, res_cam, res_xy, cams, max_iter=250):
        """l3d_optimize_lines: returns (p1p2_out[L,6], valid[L], summary[8])"""
        f64 = lambda a: np.ascontiguousarray(a, np.float64)
        p1p2, res_xy, cams = f64(p1p2), f64(res_xy), f64(cams)
        res_ptr = np.ascontiguousarray(res_ptr, np.int64); res_cam = np.ascontiguousarray(res_cam, np.int32)
        L = len(p1p2)
        out = np.zeros((L, 6), np.float64); valid = np.zeros(L, np.int32); summ = np.zeros(8, np.float64)
        self._chk(self.L.l3d_optimize_lines(self.h, L, _p(p1p2), _p(res_ptr), _p(res_cam), _p(res_xy), len(cams), _p(cams), int(max_iter),
                                            _p(out), _p(valid), _p(summ)), "l3d_optimize_lines")
        return out, valid, summ

    def fp32_peak_tflops(self) -> float:
        v = C.c_double(0)
        self._chk(self.L.l3d_fp32_peak_probe(self.h, C.byref(v)), "l3d_fp32_peak_probe")
        return v.value

    def match_dense_pairs(self, pairs, F, epi_overlap, depth_ptrs, overlap_ptrs):
        """dense contract for many view pairs in one launch; depth_ptrs / overlap_ptrs: device addresses per pair"""
        pairs = np.ascontiguousarray(pairs, np.int32).reshape(-1, 2)
        F = np.ascontiguousarray(F, np.float32).reshape(-1, 9)
        dp = (C.c_void_p * len(pairs))(*[int(x) for x in depth_ptrs])
        op = (C.c_void_p * len(pairs))(*[int(x) for x in overlap_ptrs])
        self._chk(self.L.l3d_match_dense_pairs(self.h, len(pairs), _p(pairs), _p(F), epi_overlap, dp, op), "l3d_match_dense_pairs")

    # ---- tie points (stateless: no pipeline stage changes)
    def triangulate_points(self, obs_ptr, obs_cam, obs_xy, P):
        """l3d_triangulate_points on host arrays: obs_ptr int64 [n+1] (CSR over points), obs_cam int32 [m], obs_xy float64 [m, 2],
        P float64 [cams, 3, 4].  Returns (X float64 [n, 3], valid int32 [n])."""
        ptr = np.ascontiguousarray(obs_ptr, np.int64)
        cam = np.ascontiguousarray(obs_cam, np.int32)
        xy = np.ascontiguousarray(obs_xy, np.float64).reshape(-1, 2)
        P = np.ascontiguousarray(P, np.float64).reshape(-1, 12)
        n = len(ptr) - 1
        if n < 0 or len(cam) != len(xy) or (n >= 0 and ptr[-1] != len(cam)):
            raise ValueError("obs_ptr must have n+1 entries ending at the number of observations")
        X = np.zeros((n, 3), np.float64); valid = np.zeros(n, np.int32)
        self._chk(self.L.l3d_triangulate_points(self.h, n, _p(ptr), _p(cam), _p(xy), len(P), _p(P), _p(X), _p(valid), 0),
                  "l3d_triangulate_points")
        return X, valid

    def triangulate_points_device(self, n, obs_ptr, obs_cam, obs_xy, n_cams, P, X_out, valid_out):
        """l3d_triangulate_points on device addresses; asynchronous on the context's stream"""
        self._chk(self.L.l3d_triangulate_points(self.h, n, int(obs_ptr), int(obs_cam), int(obs_xy), int(n_cams), int(P), int(X_out), int(valid_out), 1),
                  "l3d_triangulate_points")

    def median_depths(self, list_ptr, list_pts, X, valid, centres):
        """l3d_median_depths on host arrays: per camera the points list_pts[list_ptr[c]:list_ptr[c+1]] and its centre.  Returns
        (count int32 [cams], median float32 [cams])."""
        lptr = np.ascontiguousarray(list_ptr, np.int64)
        lpts = np.ascontiguousarray(list_pts, np.int32)
        X = np.ascontiguousarray(X, np.float64).reshape(-1, 3)
        valid = np.ascontiguousarray(valid, np.int32)
        Cs = np.ascontiguousarray(centres, np.float64).reshape(-1, 3)
        nc = len(lptr) - 1
        if nc != len(Cs) or len(valid) != len(X) or lptr[-1] != len(lpts):
            raise ValueError("list_ptr needs one entry per camera + 1 and must end at len(list_pts); valid needs one flag per point")
        cnt = np.zeros(nc, np.int32); med = np.zeros(nc, np.float32)
        self._chk(self.L.l3d_median_depths(self.h, nc, _p(lptr), _p(lpts), len(X), _p(X), _p(valid), _p(Cs), _p(cnt), _p(med), 0),
                  "l3d_median_depths")
        return cnt, med

    def median_depths_device(self, n_cams, list_ptr, list_pts, n_points, X, valid, centres, count_out, median_out):
        """l3d_median_depths on device addresses; asynchronous on the context's stream apart from reading list_ptr[n_cams] (a point id
        outside [0, n_points) counts as invalid)"""
        self._chk(self.L.l3d_median_depths(self.h, int(n_cams), int(list_ptr), int(list_pts), int(n_points), int(X), int(valid), int(centres),
                                           int(count_out), int(median_out), 1), "l3d_median_depths")

    # ---- lens undistortion (stateless: no pipeline stage changes)
    def undistort(self, images, K, radial=(0, 0, 0), tangential=(0, 0), out=None, lens=None):
        """Line3D::undistortImage for a list of uint8 HxW / HxWx3 images in ONE batched call.  K, radial, tangential: one camera for
        all images or one per image.  lens: instead of radial / tangential, one lens dict (lens_desc_args) or a list with one per image.
        out: optional list of preallocated outputs (any row pitch).  Returns the output arrays."""
        n = len(images)
        per = lambda v, nd: [v] * n if np.ndim(v) == nd else list(v)
        Ks, rads, tans = per(K, 2), per(radial, 1), per(tangential, 1)
        lenses = [None] * n if lens is None else [lens] * n if isinstance(lens, dict) else list(lens)
        descs, keep = (UndistortDesc * n)(), []
        outs = []
        for i, img in enumerate(images):
            a, sp = _image_rows(img)
            o = np.empty_like(a) if out is None else out[i]
            if o.shape != a.shape or o.dtype != np.uint8 or o.strides[1:] != a.strides[1:]:
                raise ValueError("output must be a uint8 array of the input's shape with packed rows")
            keep += [a, o]
            lk = dict(radial=rads[i], tangential=tans[i]) if lenses[i] is None else lens_desc_args(lenses[i])
            descs[i] = make_undistort_desc(a.shape[1], a.shape[0], 1 if a.ndim == 2 else 3, Ks[i], src=a.ctypes.data, src_pitch=sp,
                                           dst=o.ctypes.data, dst_pitch=o.strides[0], **lk)
            outs.append(o)
        self._chk(self.L.l3d_undistort_u8(self.h, n, descs, 0), "l3d_undistort_u8")
        return outs

    # ---- image preparation for line detection (stateless: no pipeline stage changes)
    def prepare_gray(self, images, max_img_width):
        """l3d_prepare_gray_u8 for a list of uint8 HxW / HxWx3 images in ONE batched call; max_img_width: one value for all images or
        one per image.  Returns the grey uint8 [out_h, out_w] arrays."""
        n = len(images)
        mws = [max_img_width] * n if np.ndim(max_img_width) == 0 else list(max_img_width)
        descs, keep, outs = (ImagePrepDesc * n)(), [], []
        for i, img in enumerate(images):
            a, sp = _image_rows(img)
            c = 1 if a.ndim == 2 else 3
            ow, oh, _ = image_prep_size(a.shape[1], a.shape[0], mws[i])
            o = np.empty((oh, ow), np.uint8)
            keep += [a, o]
            descs[i] = make_image_prep_desc(a.shape[1], a.shape[0], c, mws[i], a.ctypes.data, sp, o.ctypes.data, ow)
            outs.append(o)
        self._chk(self.L.l3d_prepare_gray_u8(self.h, n, descs, 0), "l3d_prepare_gray_u8")
        return outs

    def prepare_gray_device(self, descs):
        """l3d_prepare_gray_u8 on device addresses (a ctypes array of ImagePrepDesc); asynchronous on the context's stream"""
        self._chk(self.L.l3d_prepare_gray_u8(self.h, len(descs), descs, 1), "l3d_prepare_gray_u8")

    def undistort_device(self, descs):
        """l3d_undistort_u8 on device addresses (a ctypes array of UndistortDesc); asynchronous on the context's stream"""
        self._chk(self.L.l3d_undistort_u8(self.h, len(descs), descs, 1), "l3d_undistort_u8")

    def undistort_map(self, width, height, K, radial=(0, 0, 0), tangential=(0, 0), lens=None):
        """the fixed-point maps cv::remap takes: (map_xy int16 [h, w, 2], map_frac uint16 [h, w]); lens as in undistort"""
        lk = dict(radial=radial, tangential=tangential) if lens is None else lens_desc_args(lens)
        d = make_undistort_desc(width, height, 1, K, **lk)
        xy = np.empty((height, width, 2), np.int16)
        fr = np.empty((height, width), np.uint16)
        self._chk(self.L.l3d_undistort_map(self.h, C.byref(d), _p(xy), _p(fr), 0), "l3d_undistort_map")
        return xy, fr

    def remap(self, image, map_xy, map_frac):
        """cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) of a uint8 HxW / HxWx3 image with fixed-point maps"""
        a, sp = _image_rows(image)
        xy = np.ascontiguousarray(map_xy, np.int16)
        fr = np.ascontiguousarray(map_frac, np.uint16)
        if xy.shape != a.shape[:2] + (2,) or fr.shape != a.shape[:2]:
            raise ValueError("maps must be [h, w, 2] int16 and [h, w] uint16")
        o = np.empty(a.shape, np.uint8)
        d = make_undistort_desc(a.shape[1], a.shape[0], 1 if a.ndim == 2 else 3, np.eye(3), src=a.ctypes.data, src_pitch=sp, dst=o.ctypes.data)
        self._chk(self.L.l3d_remap_u8(self.h, C.byref(d), _p(xy), _p(fr), 0), "l3d_remap_u8")
        return o

    def match_dense(self, src_view, tgt_view, F, epi_overlap, ns, nt, nofilter=False, dev_ptrs=None):
        F = np.ascontiguousarray(F, np.float32).reshape(9)
        fn = self.L.l3d_match_dense_nofilter if nofilter else self.L.l3d_match_dense
        if dev_ptrs is not None:
            self._chk(fn(self.h, int(src_view), int(tgt_view), _p(F), epi_overlap, dev_ptrs[0], dev_ptrs[1], 1), "l3d_match_dense")
            return None
        dep = np.empty((ns, nt, 4), np.float32)
        ov = np.empty((ns, nt), np.float32)
        self._chk(fn(self.h, int(src_view), int(tgt_view), _p(F), epi_overlap, _p(dep), _p(ov), 0),
                  "l3d_match_dense")
        return dep, ov
