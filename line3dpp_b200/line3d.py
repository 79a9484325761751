"""Python face of the C++ L3DPP::Line3D mirror (include/line3d.h, csrc/line3d_host.cc) via its C wrapper.

Used by the tests and tools; the arithmetic is all in libl3d_b200.so (GPU) — nothing is computed here.
"""
from __future__ import annotations

import ctypes as C
import threading

import numpy as np

from . import capi

SEG3D_DT = np.dtype([("line", "<i4"), ("_pad", "<i4"), ("p1", "<f8", 3), ("p2", "<f8", 3)])
RESID_DT = np.dtype([("line", "<i4"), ("cam", "<u4"), ("seg", "<u4")])


class Stats(C.Structure):
    _fields_ = [(n, C.c_longlong) for n in ("view_pairs", "pair_evaluations", "matches_after_knn", "estimates", "affinity_entries",
                                            "affinity_rows", "clusters_total", "clusters_valid", "lines3D", "collinear_entries", "opt_iterations")] + \
               [(n, C.c_double) for n in ("ms_match", "ms_score", "ms_affinity", "ms_diffusion", "ms_cluster", "opt_cost_before", "opt_cost_after",
                                          "ms_gather")]


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


# l3dpp_detect_fn (include/l3dpp_capi.h): (user, gray pixels, rows, cols, detections handle) -> non-zero on success
DETECT_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.POINTER(C.c_uint8), C.c_int, C.c_int, C.c_void_p)


class Line3D:
    """addImage / matchImages / reconstruct3Dlines with the reference's argument meaning (line3D.h:80-166)."""

    def __init__(self, neighbors_by_worldpoints=True, use_gpu=True, device=0, output_folder=None, load_segments=True, max_img_width=-1,
                 devices=None, max_line_segments=3000):
        """output_folder / load_segments / max_img_width / max_line_segments: the reference's constructor arguments; with an output
        folder, add_image with no segments reads the segment cache under <output_folder>/L3D++_data/ (segment_cache_path), and
        add_image_pixels also writes it.
        devices: a list of CUDA devices in place of `device` (the first is the primary; repeats allowed): match_images splits the
        view pairs over them and gathers the matches on the primary, with the single-device result"""
        self.L = capi.lib()
        devs = np.ascontiguousarray([int(d) for d in ([device] if devices is None else devices)], np.int32)
        if len(devs) == 0:
            raise ValueError("devices must name at least one CUDA device")
        h = self.L.l3dpp_create(str(output_folder or "").encode(), int(load_segments), int(max_img_width), int(max_line_segments),
                                int(neighbors_by_worldpoints), int(use_gpu), _p(devs), len(devs))
        self.h = C.c_void_p(h)
        if not self.h:
            which = "" if devices is None else f" among {list(devices)}"
            raise capi.L3DError(f"L3DPP::Line3D: no usable CUDA device{which} (no CPU fallback)")
        self.ctx = C.c_void_p(self.L.l3dpp_ctx(self.h))

    def close(self):
        if getattr(self, "h", None):
            self.L.l3dpp_destroy(self.h)
            self.h = None

    def __del__(self):
        self.close()

    def _chk(self, rc, what):
        if rc < 0:
            raise capi.L3DError(f"{what}: {self.L.l3dpp_last_error(self.h).decode()}")
        return rc

    def add_image(self, cam, width, height, K, R, t, median_depth, wps_or_neighbors, segs=(), lens=None):
        """segs: float32 [n, 4]; empty: read the view's segment cache (see __init__).  lens: the camera's lens dict (as read_colmap
        gives it): segs are then in the distorted image and their endpoints are undistorted into K (a cached list is used as stored)"""
        lst = np.ascontiguousarray(wps_or_neighbors, np.uint32)
        segs = np.ascontiguousarray(segs, np.float32).reshape(-1, 4)
        f64 = lambda a: np.ascontiguousarray(a, np.float64)
        if lens is None:
            rc = self.L.l3dpp_add_image(self.h, int(cam), int(width), int(height), _p(f64(K)), _p(f64(R)), _p(f64(t)), float(median_depth),
                                        _p(lst), len(lst), _p(segs), len(segs))
        else:
            rc = self.L.l3dpp_add_image_lens(self.h, int(cam), int(width), int(height), _p(f64(K)), _p(f64(R)), _p(f64(t)), float(median_depth),
                                             _p(lst), len(lst), _p(_lens9(lens)), _p(segs), len(segs))
        self._chk(rc, "addImage")

    def add_image_pixels(self, cam, img, K, R, t, median_depth, wps_or_neighbors, segs=(), lens=None):
        """addImage with the image itself: img uint8 HxW (grey) or HxWx3 (channel 0 is R), any row stride.  Without segs the segment
        cache is read, or the image is prepared on the GPU and handed to the set_segment_detector function.  An exception raised by
        the detector is raised here again.  lens: the camera's lens dict; img and segs are then the distorted image and segments in
        it: the image is undistorted into K on the GPU before it is prepared, the segments' endpoints are undistorted into K."""
        a, sp = capi._image_rows(img)
        lst = np.ascontiguousarray(wps_or_neighbors, np.uint32)
        segs = np.ascontiguousarray(segs, np.float32).reshape(-1, 4)
        f64 = lambda v: np.ascontiguousarray(v, np.float64)
        errors = self.__dict__.setdefault("_detector_errors", {})      # per calling thread: the detector runs on it
        errors.pop(threading.get_ident(), None)
        if lens is None:
            rc = self.L.l3dpp_add_image_pixels(self.h, int(cam), a.ctypes.data, a.shape[0], a.shape[1], 1 if a.ndim == 2 else 3, sp, _p(f64(K)),
                                               _p(f64(R)), _p(f64(t)), float(median_depth), _p(lst), len(lst), _p(segs), len(segs))
        else:
            rc = self.L.l3dpp_add_image_pixels_lens(self.h, int(cam), a.ctypes.data, a.shape[0], a.shape[1], 1 if a.ndim == 2 else 3, sp,
                                                    _p(f64(K)), _p(f64(R)), _p(f64(t)), float(median_depth), _p(lst), len(lst),
                                                    _p(_lens9(lens)), _p(segs), len(segs))
        err = errors.pop(threading.get_ident(), None)
        if err is not None:
            raise err
        self._chk(rc, "addImage")

    def set_segment_detector(self, fn):
        """fn(gray uint8 [rows, cols]) -> detections float32 [n, 4] (x1, y1, x2, y2 in gray's coordinates), or None / False to reject
        the view; None: no detector.  It runs on the thread that called add_image_pixels, possibly on several at once."""
        if fn is None:
            cb = None
        else:
            def call(_user, gray, rows, cols, out):
                try:
                    det = fn(np.ctypeslib.as_array(gray, shape=(rows, cols)).copy())
                    if det is None or det is False:
                        return 0
                    det = np.ascontiguousarray(det, np.float32).reshape(-1, 4)
                    self.L.l3dpp_push_detections(out, _p(det), len(det))
                    return 1
                except BaseException as e:      # noqa: BLE001 - handed back to add_image_pixels
                    self.__dict__.setdefault("_detector_errors", {})[threading.get_ident()] = e
                    return 0
            cb = DETECT_FN(call)
        self._detector = cb                     # the library keeps the pointer: keep the callback alive
        self.L.l3dpp_set_segment_detector(self.h, cb, None)

    def set_line_candidates(self, cam_a, cam_b, seg_pairs):
        """Line3D::setLineCandidates: match the view pair {cam_a, cam_b} only against seg_pairs, an (n, 2) integer array of (segment of
        cam_a, segment of cam_b); empty: no matches on the pair.  Replaces the pair's earlier list; kept until clear_line_candidates"""
        a = np.asarray(seg_pairs, np.int64).reshape(-1, 2)
        if (a < 0).any() or (a > 0xFFFFFFFF).any():
            raise ValueError("segment IDs must be in [0, 2^32)")
        a = np.ascontiguousarray(a, np.uint32)
        self._chk(self.L.l3dpp_set_line_candidates(self.h, int(cam_a), int(cam_b), _p(a), len(a)), "setLineCandidates")

    def clear_line_candidates(self):
        """Line3D::clearLineCandidates: every view pair is scanned again"""
        self._chk(self.L.l3dpp_clear_line_candidates(self.h), "clearLineCandidates")

    def view_segments(self, cam):
        """float32 [n, 4]: the view's 2D segments as getSegmentCoords2D returns them"""
        n = self.L.l3dpp_view_segments(self.h, int(cam), None, 0)
        if n < 0:
            raise KeyError(cam)
        out = np.zeros((n, 4), np.float32)
        self.L.l3dpp_view_segments(self.h, int(cam), _p(out), n)
        return out

    def add_scene(self, scene):
        for i in range(scene.num_views):
            self.add_image(scene.cam_ids[i], scene.width, scene.height, scene.K[i], scene.R[i], scene.t[i], scene.median_depth[i],
                           scene.neighbors[i], scene.segs[i])

    def match_images(self, sigma_p=2.5, sigma_a=10.0, num_neighbors=10, epi_overlap=0.25, knn=10, const_reg_depth=-1.0):
        self._chk(self.L.l3dpp_match_images(self.h, sigma_p, sigma_a, num_neighbors, epi_overlap, knn, const_reg_depth), "matchImages")

    def reconstruct_3d_lines(self, visibility_t=3, perform_diffusion=False, collinearity_t=-1.0, use_ceres=False, max_iter_ceres=250):
        self._chk(self.L.l3dpp_reconstruct_opt(self.h, visibility_t, int(perform_diffusion), collinearity_t, int(use_ceres), max_iter_ceres),
                  "reconstruct3Dlines")

    # ---- dumps
    def stats(self):
        s = Stats()
        self.L.l3dpp_stats(self.h, C.byref(s))
        return {n: getattr(s, n) for n, _ in Stats._fields_}

    def pairs(self):
        n = self.L.l3dpp_get_pairs(self.h, None, 0)
        a = np.zeros((n, 2), np.int32)
        self.L.l3dpp_get_pairs(self.h, _p(a), n)
        return a

    def view_info(self, cam):
        k, md = C.c_float(0), C.c_float(0)
        self.L.l3dpp_view_info(self.h, int(cam), C.byref(k), C.byref(md))
        return k.value, md.value

    def view_matches(self, cam, kept_only):
        vi = self.L.l3dpp_view_index(self.h, int(cam))
        n = self.L.l3d_get_view_matches(self.ctx, vi, int(kept_only), None, 0)
        if n < 0:
            raise capi.L3DError("l3d_get_view_matches failed")
        a = np.zeros(n, capi.MATCH_DT)
        if n:
            self.L.l3d_get_view_matches(self.ctx, vi, int(kept_only), _p(a), n)
        return a

    def estimates(self):
        n = self.L.l3d_get_estimates(self.ctx, None, None, 0)
        best, p = np.zeros(max(n, 0), capi.MATCH_DT), np.zeros((max(n, 0), 6), np.float64)
        if n > 0:
            self.L.l3d_get_estimates(self.ctx, _p(best), _p(p), n)
        return best, p

    def ctx_collinear(self, view_index, nseg):
        """View::collin_ of the view_index-th added view as CSR (row_ptr, idx), straight from the C ABI"""
        row_ptr = np.zeros(nseg + 1, np.int64)
        n = self.L.l3d_get_collinear(self.ctx, int(view_index), _p(row_ptr), None, 0)
        if n < 0:
            raise capi.L3DError("l3d_get_collinear failed")
        idx = np.zeros(max(int(n), 1), np.int32)
        if n > 0:
            self.L.l3d_get_collinear(self.ctx, int(view_index), _p(row_ptr), _p(idx), n)
        return row_ptr, idx[:int(n)]

    def affinity(self, raw=False):
        n = self.L.l3dpp_get_affinity(self.h, int(raw), None, None, None, 0)
        ei, ej, ew = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.float32)
        if n:
            self.L.l3dpp_get_affinity(self.h, int(raw), _p(ei), _p(ej), _p(ew), n)
        return ei, ej, ew

    def local2global(self):
        n = self.L.l3dpp_get_local2global(self.h, None, 0)
        a = np.zeros((n, 2), np.uint32)
        if n:
            self.L.l3dpp_get_local2global(self.h, _p(a), n)
        return a

    def segments3d(self):
        n = self.L.l3dpp_get_segments3d(self.h, None, 0)
        a = np.zeros(n, SEG3D_DT)
        if n:
            self.L.l3dpp_get_segments3d(self.h, _p(a), n)
        return a

    def residuals(self):
        n = self.L.l3dpp_get_residuals(self.h, None, 0)
        a = np.zeros(n, RESID_DT)
        if n:
            self.L.l3dpp_get_residuals(self.h, _p(a), n)
        return a

    def save_txt(self, folder):
        self._chk(self.L.l3dpp_save_txt(self.h, folder.encode()), "save3DLinesAsTXT")

    def lines(self):
        """get3Dlines() with every field, in the layout read_lines_bin returns"""
        return _lines_from_handle(self.L, self.L.l3dpp_lines_handle(self.h))

    def save_bin(self, folder):
        """save3DLinesAsBIN: <folder>/<createOutputFilename()>.bin; nothing is written (and L3DError is raised) without 3D lines"""
        self._chk(self.L.l3dpp_save_bin(self.h, str(folder).encode()), "save3DLinesAsBIN")

    def output_filename(self):
        buf = C.create_string_buffer(1024)
        self._chk(self.L.l3dpp_output_filename(self.h, buf, 1024), "createOutputFilename")
        return buf.value.decode()


# ---- the reference's binary files (include/line3d_io.h, csrc/line3d_bin.cc); host only, no GPU needed
LINE_DT = np.dtype([("nseg", "<i4"), ("nres", "<i4"), ("reference_view", "<u4"), ("_pad", "<i4")])
BIN_SEG_DT = np.dtype([("line", "<i4"), ("valid", "<i4"), ("length", "<f4"), ("_pad", "<i4"), ("p1", "<f8", 3), ("p2", "<f8", 3),
                       ("dir", "<f8", 3)])


def read_lines_bin(path):
    """read3DLinesBIN: a .bin result file as numpy arrays.  Returns dict(lines: LINE_DT [L] (segment / residual counts, reference
    view), clusters: BIN_SEG_DT [L] (each cluster's own 3D line), segments: BIN_SEG_DT [S], residuals: RESID_DT [R]); segments and
    residuals of line i are consecutive and carry line = i.  Raises L3DError with the reader's message on a malformed file."""
    L = capi.lib()
    err = C.create_string_buffer(1024)
    h = L.l3dpp_bin_open(str(path).encode(), err, 1024)
    if not h:
        raise capi.L3DError(err.value.decode())
    return _lines_from_handle(L, h)


def _lines_from_handle(L, h):
    """the arrays of a std::vector<FinalLine3D> handle (l3dpp_bin_*); closes the handle"""
    try:
        nl, ns, nr = C.c_longlong(), C.c_longlong(), C.c_longlong()
        L.l3dpp_bin_sizes(h, C.byref(nl), C.byref(ns), C.byref(nr))
        out = dict(lines=np.zeros(nl.value, LINE_DT), clusters=np.zeros(nl.value, BIN_SEG_DT), segments=np.zeros(ns.value, BIN_SEG_DT),
                   residuals=np.zeros(nr.value, RESID_DT))
        L.l3dpp_bin_get(h, _p(out["lines"]), _p(out["clusters"]), _p(out["segments"]), _p(out["residuals"]))
    finally:
        L.l3dpp_bin_close(h)
    return out


def write_lines_bin(path, d):
    """write3DLinesBIN of a dict as read_lines_bin returns it"""
    lines = np.ascontiguousarray(d["lines"], LINE_DT)
    clusters = np.ascontiguousarray(d["clusters"], BIN_SEG_DT)
    segs = np.ascontiguousarray(d["segments"], BIN_SEG_DT)
    res = np.ascontiguousarray(d["residuals"], RESID_DT)
    if len(clusters) != len(lines) or lines["nseg"].sum() != len(segs) or lines["nres"].sum() != len(res):
        raise ValueError("clusters must have one entry per line, and the per-line counts must add up to the segment / residual arrays")
    err = C.create_string_buffer(1024)
    if capi.lib().l3dpp_bin_write(str(path).encode(), len(lines), _p(lines), _p(clusters), _p(segs), _p(res), err, 1024) != 0:
        raise capi.L3DError(err.value.decode())


def read_segment_cache(path):
    """readSegmentCache: a view's cached 2D segments as float32 [n, 4] (x1, y1, x2, y2)"""
    L = capi.lib()
    err = C.create_string_buffer(1024)
    h = L.l3dpp_segcache_open(str(path).encode(), err, 1024)
    if not h:
        raise capi.L3DError(err.value.decode())
    try:
        out = np.zeros((L.l3dpp_segcache_count(h), 4), np.float32)
        L.l3dpp_segcache_get(h, _p(out))
    finally:
        L.l3dpp_segcache_close(h)
    return out


def write_segment_cache(path, segs):
    """writeSegmentCache of float32 [n, 4] segments"""
    segs = np.ascontiguousarray(segs, np.float32).reshape(-1, 4)
    err = C.create_string_buffer(1024)
    if capi.lib().l3dpp_segcache_write(str(path).encode(), _p(segs), len(segs), err, 1024) != 0:
        raise capi.L3DError(err.value.decode())


def segment_cache_path(output_folder, cam, width, height, max_img_width=-1):
    """segmentCachePath: <output_folder>/L3D++_data/segments_L3D++_<cam>_<w>x<h>_3000.bin"""
    buf = C.create_string_buffer(4096)
    n = capi.lib().l3dpp_segcache_path(str(output_folder).encode(), int(cam), int(width), int(height), int(max_img_width), buf, 4096)
    if n < 0:
        raise ValueError("path too long")
    return buf.value.decode()


# ---- SfM models (include/line3d_io.h, csrc/line3d_sfm.cc); host only except read_pix4d, which triangulates on a GPU
def _worldpoints(get, h, i, n):
    """the n world point ids of camera i through l3dpp_nvm_worldpoints / l3dpp_sfm_worldpoints"""
    w = np.zeros(max(n, 1), np.uint32)
    if get(h, i, _p(w), n) != n:
        raise capi.L3DError(f"world point count of camera {i} changed")
    return w[:n]


def read_nvm(path):
    """readNVM: the cameras of an NVM_V3 file as dicts (image, focal, distortion, R, t, C, median_depth, worldpoints).  Raises L3DError
    on a malformed model."""
    L = capi.lib()
    err = C.create_string_buffer(4096)
    h = L.l3dpp_nvm_open(str(path).encode(), err, 4096)
    if not h:
        raise capi.L3DError(err.value.decode(errors="replace"))
    cams = []
    try:
        for i in range(L.l3dpp_nvm_num_cameras(h)):
            R, t, Cc = np.zeros(9), np.zeros(3), np.zeros(3)
            f, d, md, nw = C.c_float(), C.c_float(), C.c_float(), C.c_int()
            name = C.create_string_buffer(4096)
            if L.l3dpp_nvm_camera(h, i, _p(R), _p(t), _p(Cc), C.byref(f), C.byref(d), C.byref(md), C.byref(nw), name, 4096) != 0:
                raise capi.L3DError(f"no camera {i}")
            cams.append(dict(image=name.value.decode(errors="replace"), focal=np.float32(f.value), distortion=np.float32(d.value), R=R.reshape(3, 3),
                             t=t, C=Cc, median_depth=np.float32(md.value), worldpoints=_worldpoints(L.l3dpp_nvm_worldpoints, h, i, nw.value)))
    finally:
        L.l3dpp_nvm_close(h)
    return cams


def _sfm_cameras(L, h, lenses=False):
    """the cameras of an l3dpp_sfm_* handle as dicts (id, image, has_K, K, focal, R, t, C, radial, tangential, median_depth, worldpoints,
    and with lenses the lens dict {model, k[6], p[2]} of L3DPP::LensDistortion); closes it"""
    cams = []
    try:
        for i in range(L.l3dpp_sfm_num_cameras(h)):
            head, K, R, t, Cc, dist = np.zeros(5), np.zeros(9), np.zeros(9), np.zeros(3), np.zeros(3), np.zeros(5)
            name = C.create_string_buffer(4096)
            if L.l3dpp_sfm_camera(h, i, _p(head), _p(K), _p(R), _p(t), _p(Cc), _p(dist), name, 4096) != 0:
                raise capi.L3DError(f"no camera {i}")
            cams.append(dict(id=int(head[0]), image=name.value.decode(errors="replace"), has_K=bool(head[1]), K=K.reshape(3, 3),
                             focal=np.float32(head[2]), R=R.reshape(3, 3), t=t, C=Cc, radial=dist[:3].copy(), tangential=dist[3:].copy(),
                             median_depth=np.float32(head[3]), worldpoints=_worldpoints(L.l3dpp_sfm_worldpoints, h, i, int(head[4]))))
            if lenses:
                lens = np.zeros(9)
                if L.l3dpp_sfm_lens(h, i, _p(lens)) != 0:
                    raise capi.L3DError(f"no lens for camera {i}")
                cams[-1]["lens"] = dict(model=int(lens[0]), k=lens[1:7].copy(), p=lens[7:9].copy())
    finally:
        L.l3dpp_sfm_close(h)
    return cams


# the model kinds of l3dpp_sfm_open (L3DPP_SFM_* of include/l3dpp_capi.h)
SFM_BUNDLER, SFM_COLMAP, SFM_MAVMAP, SFM_OPENMVG, SFM_PIX4D, SFM_COLMAP_LENSES = range(6)


def _read_sfm(kind, path, aux=""):
    L = capi.lib()
    err = C.create_string_buffer(4096)
    h = L.l3dpp_sfm_open(int(kind), str(path).encode(), str(aux).encode(), err, 4096)
    if not h:
        raise capi.L3DError(err.value.decode(errors="replace"))
    return _sfm_cameras(L, h, lenses=kind == SFM_COLMAP_LENSES)


def read_bundler(bundle_file, image_list=""):
    """readBundler: the cameras of a bundle.rd.out (focal only, has_K False; names from the optional image list).  Raises L3DError on
    a malformed model."""
    return _read_sfm(SFM_BUNDLER, bundle_file, image_list)


def read_colmap(sfm_folder, lenses=True):
    """readColmap: the cameras of a COLMAP model (cameras/images/points3D .txt, or else .bin).  With lenses each has a `lens` dict
    {model: capi.LENS_RADTAN | capi.LENS_FISHEYE, k: k1..k6, p: p1, p2} for undistort_image; without, fisheye cameras are rejected.
    Raises L3DError on a malformed model."""
    return _read_sfm(SFM_COLMAP_LENSES if lenses else SFM_COLMAP, sfm_folder)


def _lens9(lens):
    """a lens dict as L3DPP::LensDistortion's 9 doubles: model, k[6], p[2]"""
    k = [float(v) for v in lens.get("k", ())] + [0.0] * 6
    pp = [float(v) for v in lens.get("p", ())] + [0.0] * 2
    return np.array([float(lens.get("model", capi.LENS_RADTAN))] + k[:6] + pp[:2], np.float64)


def undistort_image(img, K, lens, new_K=None, out_size=None, device=0):
    """Line3D::undistortImage(in, out, lens, K[, newK, out_width, out_height]) of a uint8 HxW / HxWx3 image on GPU `device`; lens as
    read_colmap gives it.  new_K: the output's camera matrix (None: K), e.g. from optimal_new_camera_matrix or
    fisheye_new_camera_matrix; out_size: the output's (width, height) (None: the image's)"""
    a = np.ascontiguousarray(img, np.uint8)
    if a.ndim not in (2, 3) or (a.ndim == 3 and a.shape[2] != 3):
        raise ValueError("image must be uint8 HxW or HxWx3")
    Kd = np.ascontiguousarray(K, np.float64).reshape(9)
    nK = np.zeros(9) if new_K is None else np.ascontiguousarray(new_K, np.float64).reshape(9)
    ow, oh = (0, 0) if out_size is None else (int(out_size[0]), int(out_size[1]))
    out = np.empty(((oh, ow) if out_size is not None and ow >= 1 and oh >= 1 else a.shape[:2]) + a.shape[2:], np.uint8)
    L = capi.lib()
    rc = L.l3dpp_undistort_image_newk(_p(a), _p(out), a.shape[0], a.shape[1], 1 if a.ndim == 2 else 3, _p(_lens9(lens)), _p(Kd), _p(nK), oh, ow,
                                      int(device))
    if rc == -1:
        raise ValueError("undistort_image: an image, lens, new K or size l3d_undistort_u8 rejects")
    if rc != 0:
        raise capi.L3DError("undistort_image: no usable CUDA device or a CUDA failure")
    return out


def undistort_points(pts, K, lens, new_K=None, device=0):
    """Line3D::undistortPoints on GPU `device`: cv2.undistortPoints(pts, K, D, None, new_K) for a radtan lens dict and
    cv2.fisheye.undistortPoints(pts, K, D, R=I, P=new_K) for a fisheye one (DESIGN.md §4a).  pts: float32 (x, y) pairs of any shape
    [..., 2] (segments [n, 4] are two points each); new_K None: K.  Returns float32 points of pts' shape, in pixels of new_K."""
    return undistort_points_batch([(pts, K, lens, new_K)], device)[0]


def undistort_points_batch(sets, device=0):
    """the batched Line3D::undistortPoints: a list of (pts, K, lens, new_K) sets undistorted in one launch; returns one array per set"""
    arrs = [np.asarray(s[0], np.float32) for s in sets]
    if any(a.size % 2 for a in arrs):
        raise ValueError("undistort_points: points are (x, y) pairs")
    cat = lambda parts, dt: np.ascontiguousarray(np.concatenate(parts) if parts else np.zeros(0, dt), dt)
    xy = cat([a.reshape(-1) for a in arrs], np.float32)
    counts = np.array([a.size // 2 for a in arrs], np.int64)
    lens9 = cat([_lens9(s[2]) for s in sets], np.float64)
    Ks = cat([np.asarray(s[1], np.float64).reshape(9) for s in sets], np.float64)
    nKs = cat([np.zeros(9) if s[3] is None else np.asarray(s[3], np.float64).reshape(9) for s in sets], np.float64)
    err = C.create_string_buffer(512)
    rc = capi.lib().l3dpp_undistort_points(_p(xy), _p(counts), len(sets), _p(lens9), _p(Ks), _p(nKs), int(device), err, 512)
    if rc == -1:
        raise ValueError(err.value.decode())
    if rc != 0:
        raise capi.L3DError(err.value.decode())
    offs = np.concatenate([[0], np.cumsum([a.size for a in arrs])]).astype(np.int64)
    return [xy[offs[i]:offs[i + 1]].reshape(a.shape).copy() for i, a in enumerate(arrs)]


def optimal_new_camera_matrix(K, lens, image_size, alpha, new_size=None, center_principal_point=False):
    """Line3D::getOptimalNewCameraMatrix, i.e. cv2.getOptimalNewCameraMatrix(K, D, image_size, alpha, new_size, centerPrincipalPoint)
    for a radtan lens dict: (new K 3x3, valid-pixel ROI (x, y, width, height)).  Sizes are (width, height); host only"""
    newK, roi = np.zeros(9), np.zeros(4, np.int32)
    nw, nh = (0, 0) if new_size is None else (int(new_size[0]), int(new_size[1]))
    rc = capi.lib().l3dpp_optimal_new_camera_matrix(_p(np.ascontiguousarray(K, np.float64).reshape(9)), _p(_lens9(lens)), int(image_size[0]),
                                                    int(image_size[1]), float(alpha), nw, nh, int(bool(center_principal_point)), _p(newK), _p(roi))
    if rc != 0:
        raise ValueError("optimal_new_camera_matrix: a fisheye lens, a size below 1 or a bad camera matrix")
    return newK.reshape(3, 3), tuple(int(v) for v in roi)


def fisheye_new_camera_matrix(K, lens, image_size, balance=0.0, new_size=None, fov_scale=1.0):
    """Line3D::estimateNewCameraMatrixForUndistortRectify, i.e. cv2.fisheye.estimateNewCameraMatrixForUndistortRectify(K, D,
    image_size, I, balance=, new_size=, fov_scale=) for a fisheye lens dict: the new K 3x3.  Sizes are (width, height); host only"""
    newK = np.zeros(9)
    nw, nh = (0, 0) if new_size is None else (int(new_size[0]), int(new_size[1]))
    rc = capi.lib().l3dpp_fisheye_new_camera_matrix(_p(np.ascontiguousarray(K, np.float64).reshape(9)), _p(_lens9(lens)), int(image_size[0]),
                                                    int(image_size[1]), float(balance), nw, nh, float(fov_scale), _p(newK))
    if rc != 0:
        raise ValueError("fisheye_new_camera_matrix: a radtan lens, a size below 1 or a bad camera matrix")
    return newK.reshape(3, 3)


def jpeg_size(path):
    """readJPEGSize: (width, height) of imread(path, IMREAD_GRAYSCALE)'s output, after EXIF orientation; headers only, no GPU.  Raises
    L3DError naming the reason for a file that cannot be read or is outside the supported subset."""
    w, h = C.c_int(), C.c_int()
    err = C.create_string_buffer(4096)
    if capi.lib().l3dpp_jpeg_size(str(path).encode(), C.byref(w), C.byref(h), err, 4096) != 0:
        raise capi.L3DError(err.value.decode(errors="replace"))
    return w.value, h.value


def read_jpeg_gray(path_or_paths, device=0, errors=None):
    """readJPEGGray / readJPEGsGray: imread(path, IMREAD_GRAYSCALE) as uint8 [h, w], decoded on GPU `device`; a list of paths is one
    batched decode and gives a list.  A file that fails raises L3DError with its message, unless a list `errors` is given: then every
    failed file's entry is None, and errors receives one message per file ("" for the decoded ones)."""
    return _read_gray("jpegs", path_or_paths, device, errors)


def png_size(path):
    """readPNGSize: jpeg_size for a PNG file"""
    return _size(capi.lib().l3dpp_png_size, path)


def read_png_gray(path_or_paths, device=0, errors=None):
    """readPNGGray / readPNGsGray: read_jpeg_gray for PNG files"""
    return _read_gray("pngs", path_or_paths, device, errors)


def image_size(path):
    """readImageSize: jpeg_size or png_size, chosen by the file's signature"""
    return _size(capi.lib().l3dpp_image_size, path)


def read_image_gray(path_or_paths, device=0, errors=None):
    """readImageGray / readImagesGray: read_jpeg_gray for JPEG and PNG files alike, each chosen by its signature; a mixed list is one
    JPEG batch and one PNG batch.  Any other file fails with the reason."""
    return _read_gray("images", path_or_paths, device, errors)


def _size(fn, path):
    w, h = C.c_int(), C.c_int()
    err = C.create_string_buffer(4096)
    if fn(str(path).encode(), C.byref(w), C.byref(h), err, 4096) != 0:
        raise capi.L3DError(err.value.decode(errors="replace"))
    return w.value, h.value


def _read_gray(kind, path_or_paths, device, errors):
    single = isinstance(path_or_paths, (str, bytes)) or hasattr(path_or_paths, "__fspath__")
    paths = [path_or_paths] if single else list(path_or_paths)
    L = capi.lib()
    read, image, close = (getattr(L, f"l3dpp_{kind}_{f}") for f in ("read", "image", "close"))
    arr = (C.c_char_p * len(paths))(*[str(p).encode() for p in paths])
    h = read(arr, len(paths), int(device))
    outs, msgs = [], []
    try:
        for i in range(len(paths)):
            w, ht = C.c_int(), C.c_int()
            err = C.create_string_buffer(4096)
            if image(h, i, C.byref(w), C.byref(ht), None, 0, err, 4096) != 0:
                outs.append(None)
                msgs.append(err.value.decode(errors="replace"))
                continue
            o = np.empty((ht.value, w.value), np.uint8)
            image(h, i, C.byref(w), C.byref(ht), _p(o), o.size, err, 4096)
            outs.append(o)
            msgs.append("")
    finally:
        close(h)
    if errors is not None:
        errors[:] = msgs
    elif any(msgs):
        raise capi.L3DError("; ".join(m for m in msgs if m))
    return outs[0] if single else outs


def read_mavmap(path):
    """readMavmap: the cameras of a mavmap result file (no world points; see sequential_neighbors).  Raises L3DError on malformed input."""
    return _read_sfm(SFM_MAVMAP, path)


def read_openmvg(sfm_data_json):
    """readOpenMVG: the cameras of an OpenMVG sfm_data.json with world-point lists and median depths"""
    return _read_sfm(SFM_OPENMVG, sfm_data_json)


def read_pix4d(params_folder, project_prefix):
    """readPix4D: the cameras of a Pix4D project; its tie points are triangulated on CUDA device 0 (L3DError without one)"""
    return _read_sfm(SFM_PIX4D, params_folder, project_prefix)


def sequential_neighbors(i, n_cams, num_neighbors):
    """sequentialNeighbors: the mavmap frontend's neighbour list of camera i"""
    out = np.zeros(max(int(num_neighbors), 1), np.uint32)
    n = capi.lib().l3dpp_sequential_neighbors(int(i), int(n_cams), int(num_neighbors), _p(out), len(out))
    return out[:n].tolist()


def pose_neighbors(cam_ids, K, R, t, widths, heights, median_depths, num_neighbors=10, gx=32, gy=24, device=0):
    """poseNeighbors (include/line3d_io.h): visual neighbours from camera poses alone, for add_image with neighbors_by_worldpoints=False.
    K (n, 3, 3), R (n, 3, 3), t (n, 3) with x_cam = R X + t; widths, heights, median_depths one value or one per view.  Returns one
    uint32 array of neighbour camIDs (ascending) per view.  Raises L3DError naming the view for the inputs l3d_pose_neighbors rejects."""
    ctx = capi.Context(device)
    try:
        return ctx.pose_neighbors(capi.make_pose_views(cam_ids, K, R, t, widths, heights, median_depths), num_neighbors, gx, gy)[0]
    finally:
        ctx.close()


def rotation_from_rpy(roll, pitch, yaw):
    """Line3D::rotationFromRPY"""
    R = np.zeros(9)
    capi.lib().l3dpp_rotation_from_rpy(roll, pitch, yaw, _p(R))
    return R.reshape(3, 3)


def decompose_projection_matrix(P):
    """Line3D::decomposeProjectionMatrix of a 3x4 P: (K, R, t)"""
    P = np.ascontiguousarray(P, np.float64).reshape(12)
    K, R, t = np.zeros(9), np.zeros(9), np.zeros(3)
    capi.lib().l3dpp_decompose_projection(_p(P), _p(K), _p(R), _p(t))
    return K.reshape(3, 3), R.reshape(3, 3), t
