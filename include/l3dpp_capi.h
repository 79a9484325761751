/* include/l3dpp_capi.h — the C wrapper of the host library (L3DPP::Line3D and the file readers and writers of include/line3d_io.h),
 * exported by libl3d_b200.so next to the C ABI of include/l3d_capi.h.  It serves the package's Python layer and its tests; programs
 * that embed the library use the C++ headers (include/line3d.h, include/line3d_io.h) or include/l3d_capi.h.
 *
 * Conventions: a Line3D, a model or a result file is an opaque handle (void*) until its *_close / l3dpp_destroy; arrays are caller-owned;
 * `err`, `name` and `buf` are caller buffers of `errcap` / `namecap` / `cap` bytes that receive a NUL-terminated, possibly truncated
 * message or string.  Functions that return a count return the full count even when it exceeds the capacity given. */
#ifndef L3DPP_CAPI_H_
#define L3DPP_CAPI_H_
#ifdef __cplusplus
extern "C" {
#endif

/* ---- structs the wrappers fill or read */
/* L3DPP::Line3DStats (include/line3d.h) */
typedef struct {
    long long view_pairs, pair_evaluations, matches_after_knn, estimates, affinity_entries, affinity_rows, clusters_total,
        clusters_valid, lines3D, collinear_entries, opt_iterations;
    double ms_match, ms_score, ms_affinity, ms_diffusion, ms_cluster, opt_cost_before, opt_cost_after, ms_gather;
} l3dpp_stats_block;
/* one 3D segment of get3Dlines() and the index of its line */
typedef struct { int line; int pad; double p1[3], p2[3]; } l3dpp_seg3d;
/* one residual (2D segment) of a line's cluster */
typedef struct { int line; unsigned int cam, seg; } l3dpp_residual;
/* the .bin result file: per line its segment / residual counts and reference view */
typedef struct { int nseg, nres; unsigned int reference_view; int pad; } l3dpp_bin_line;
/* a Segment3D as the .bin file holds it */
typedef struct { int line, valid; float length; int pad; double p1[3], p2[3], dir[3]; } l3dpp_bin_seg;
typedef l3dpp_residual l3dpp_bin_res;

/* ---- callbacks */
/* Line3D::SegmentDetectorFn in C terms: detect segments in the prepared grey image (rows x cols, packed) and hand them over with
 * l3dpp_push_detections(out, ...); non-zero on success */
typedef int (*l3dpp_detect_fn)(void* user, const unsigned char* gray, int rows, int cols, void* out);
/* Line3D::MatchExchangeFn (include/line3d.h, setShard) */
typedef int (*l3dpp_exchange_fn)(void* user, void* counts_dev, void* recs_dev, const long long* row_bounds, int world, int knn);

/* ---- L3DPP::Line3D (csrc/line3d_host.cc) */
/* the Line3D constructor on devices[0..num_devices) (devices[0] is the primary); NULL without a usable CUDA device */
void* l3dpp_create(const char* output_folder, int load_segments, int max_img_width, unsigned int max_line_segments,
                   int neighbors_by_worldpoints, int use_gpu, const int* devices, int num_devices);
void l3dpp_destroy(void* h);
/* the message of the last failed call; "" when it succeeded.  Calls returning int fail with -1 */
const char* l3dpp_last_error(void* h);
/* the primary device's l3d_ctx (include/l3d_capi.h), for the l3d_get_* dumps */
void* l3dpp_ctx(void* h);
int l3dpp_add_image(void* h, unsigned int cam, int w, int hgt, const double* K, const double* R, const double* t, float median_depth,
                    const unsigned int* list, int nlist, const float* segs, int nseg);
/* addImage with an image: rows x cols, 1 or 3 channels, row step in bytes; nseg == 0: no segments given */
int l3dpp_add_image_pixels(void* h, unsigned int cam, const unsigned char* pixels, int rows, int cols, int channels, long long step, const double* K,
                           const double* R, const double* t, float median_depth, const unsigned int* list, int nlist, const float* segs, int nseg);
/* the addImage overloads with a lens (include/line3d.h): lens9 = model, k[6], p[2]; the image and the segments are in the distorted image */
int l3dpp_add_image_lens(void* h, unsigned int cam, int w, int hgt, const double* K, const double* R, const double* t, float median_depth,
                         const unsigned int* list, int nlist, const double* lens9, const float* segs, int nseg);
int l3dpp_add_image_pixels_lens(void* h, unsigned int cam, const unsigned char* pixels, int rows, int cols, int channels, long long step,
                                const double* K, const double* R, const double* t, float median_depth, const unsigned int* list, int nlist,
                                const double* lens9, const float* segs, int nseg);
/* the detector of l3dpp_add_image_pixels (NULL: none); the library keeps fn and user */
int l3dpp_set_segment_detector(void* h, l3dpp_detect_fn fn, void* user);
/* appends n detections (x1, y1, x2, y2) to the `out` a detector was given; any number of calls */
void l3dpp_push_detections(void* out, const float* xy4, long long n);
int l3dpp_match_images(void* h, float sp, float sa, unsigned int nn, float epi, int knn, float crd);
int l3dpp_reconstruct_opt(void* h, unsigned int vis, int diffusion, float collin, int use_ceres, unsigned int max_iter);
int l3dpp_set_shard(void* h, int rank, int world, l3dpp_exchange_fn fn, void* user);
/* Line3D::setLineCandidates: seg_pairs[2 * n] = (segment of cam_a, segment of cam_b) per correspondence */
int l3dpp_set_line_candidates(void* h, unsigned int cam_a, unsigned int cam_b, const unsigned int* seg_pairs, long long n);
/* Line3D::clearLineCandidates */
int l3dpp_clear_line_candidates(void* h);
int l3dpp_stats(void* h, l3dpp_stats_block* out);
/* the view index of a camID after matchImages, or -1 */
int l3dpp_view_index(void* h, unsigned int cam);
/* -1 for an unknown camID */
int l3dpp_view_info(void* h, unsigned int cam, float* k, float* md);
/* the 2D segments of a view through getSegmentCoords2D: out[cap * 4]; returns the view's segment count (-1 for an unknown camID) */
long long l3dpp_view_segments(void* h, unsigned int cam, float* out, long long cap);
/* (src cam, tgt cam) in match order */
int l3dpp_get_pairs(void* h, int* out, int cap);
/* the affinity matrix after (raw == 0) or before (raw != 0) diffusion */
long long l3dpp_get_affinity(void* h, int raw, int* ei, int* ej, float* ew, long long cap);
/* (camID, segID) per local id */
int l3dpp_get_local2global(void* h, unsigned int* cam_seg, int cap);
long long l3dpp_get_segments3d(void* h, l3dpp_seg3d* out, long long cap);
long long l3dpp_get_residuals(void* h, l3dpp_residual* out, long long cap);
/* get3Dlines() as a handle of the l3dpp_bin_* functions: every field, for comparison with a .bin file */
void* l3dpp_lines_handle(void* h);
/* test hook for the cluster -> 3D segment tail: findCollinearSegments(cluster) (line3D.cc:2342-2452) on an explicit cluster
 * (line end points + (camID, segID) residuals of views added with addImage).  Returns the number of 3D segments. */
int l3dpp_collinear_from_cluster(void* h, const double* p1p2, int nres, const unsigned int* cams, const unsigned int* segs, double* out6, int cap);
/* test hook for the writers: replace the result by explicit lines (segments: 6 doubles each; residuals: camID, segID of added views) */
int l3dpp_set_lines(void* h, int nlines, const int* nseg, const double* segs6, const int* nres, const unsigned int* res_cam, const unsigned int* res_seg);
int l3dpp_save_txt(void* h, const char* folder);
int l3dpp_save_bin(void* h, const char* folder);
int l3dpp_save_obj(void* h, const char* folder);
int l3dpp_save_stl(void* h, const char* folder);
/* createOutputFilename into buf; returns its length, or -1 if it does not fit */
int l3dpp_output_filename(void* h, char* buf, int cap);
/* detectLineSegments' post-processing alone (no GPU): out[cap * 4]; returns the number of segments kept */
long long l3dpp_filter_detections(const float* det, long long n, int w, int h, int w_p, int h_p, unsigned int max_segments, float* out, long long cap);
/* Line3D::undistortImage on a packed image; K row-major, radial[3], tangential[2].  0, -1 (std::invalid_argument) or -2 (std::runtime_error) */
int l3dpp_undistort_image(const unsigned char* src, unsigned char* dst, int rows, int cols, int channels, const double* radial, const double* tangential,
                          const double* K);
/* the LensDistortion overload on CUDA device `device` (the thread's current device is restored); lens = model, k[6], p[2] as 9 doubles */
int l3dpp_undistort_image_lens(const unsigned char* src, unsigned char* dst, int rows, int cols, int channels, const double* lens9, const double* K,
                               int device);
/* the overload with a new camera matrix (newK row-major, all zero: K) and output size (out_rows = out_cols = 0: rows x cols); dst holds
 * out_rows x out_cols x channels (rows x cols x channels for 0, 0).  Same returns */
int l3dpp_undistort_image_newk(const unsigned char* src, unsigned char* dst, int rows, int cols, int channels, const double* lens9, const double* K,
                               const double* newK, int out_rows, int out_cols, int device);
/* Line3D::undistortPoints of n point sets in one launch on CUDA device `device` (the thread's current device is restored), in place: set i
 * is counts[i] (x, y) pairs of xy, following set i - 1, with lens9[9 i..] (model, k[6], p[2]), K[9 i..] and newK[9 i..] (row-major; newK
 * NULL or a set's nine zeros: its K).  0, -1 (std::invalid_argument) or -2 (std::runtime_error), with the message in err */
int l3dpp_undistort_points(float* xy, const long long* counts, int n, const double* lens9, const double* K, const double* newK, int device, char* err,
                           int errcap);
/* Line3D::getOptimalNewCameraMatrix: newK[9] row-major, roi[4] = x, y, width, height.  0, or -1 (std::invalid_argument); no GPU used */
int l3dpp_optimal_new_camera_matrix(const double* K, const double* lens9, int width, int height, double alpha, int new_width, int new_height,
                                    int center_principal_point, double* newK, int* roi);
/* Line3D::estimateNewCameraMatrixForUndistortRectify: newK[9] row-major.  0, or -1 (std::invalid_argument); no GPU used */
int l3dpp_fisheye_new_camera_matrix(const double* K, const double* lens9, int width, int height, double balance, int new_width, int new_height,
                                    double fov_scale, double* newK);

/* ---- JPEG files (csrc/line3d_jpeg.cc) */
/* readJPEGSize: imread(IMREAD_GRAYSCALE)'s size; 0, or -1 with the reason in err.  No GPU */
int l3dpp_jpeg_size(const char* path, int* width, int* height, char* err, int errcap);
/* readJPEGsGray of n files on CUDA device cuda_device: a handle for l3dpp_jpegs_image (never NULL; failures are per file) */
void* l3dpp_jpegs_read(const char* const* paths, int n, int cuda_device);
void l3dpp_jpegs_close(void* h);
/* file i of the batch: its size, and its packed grey pixels into out[cap] when cap >= width * height; -1 with the file's error in err */
int l3dpp_jpegs_image(void* h, int i, int* width, int* height, unsigned char* out, long long cap, char* err, int errcap);

/* ---- PNG files, and JPEG or PNG by signature (csrc/line3d_png.cc) */
/* readPNGSize: imread(IMREAD_GRAYSCALE)'s size; 0, or -1 with the reason in err.  No GPU */
int l3dpp_png_size(const char* path, int* width, int* height, char* err, int errcap);
/* readPNGsGray of n files on CUDA device cuda_device: a handle for l3dpp_pngs_image (never NULL; failures are per file) */
void* l3dpp_pngs_read(const char* const* paths, int n, int cuda_device);
void l3dpp_pngs_close(void* h);
/* file i of the batch: its size, and its packed grey pixels into out[cap] when cap >= width * height; -1 with the file's error in err */
int l3dpp_pngs_image(void* h, int i, int* width, int* height, unsigned char* out, long long cap, char* err, int errcap);
/* readImageSize / readImagesGray: the same for JPEG and PNG files, chosen by each file's signature */
int l3dpp_image_size(const char* path, int* width, int* height, char* err, int errcap);
void* l3dpp_images_read(const char* const* paths, int n, int cuda_device);
void l3dpp_images_close(void* h);
int l3dpp_images_image(void* h, int i, int* width, int* height, unsigned char* out, long long cap, char* err, int errcap);

/* ---- .nvm models (csrc/line3d_sfm.cc) */
void* l3dpp_nvm_open(const char* path, char* err, int errcap);
void l3dpp_nvm_close(void* h);
int l3dpp_nvm_num_cameras(void* h);
int l3dpp_nvm_camera(void* h, int i, double* R9, double* t3, double* C3, float* focal, float* distortion, float* median_depth, int* num_wps,
                     char* name, int namecap);
int l3dpp_nvm_worldpoints(void* h, int i, unsigned int* out, int cap);
void l3dpp_intrinsics_from_focal(float focal, int w, int h, double* K9);

/* ---- the other SfM models (csrc/line3d_sfm.cc) */
#define L3DPP_SFM_BUNDLER 0         /* path = the bundle file, aux = the image list */
#define L3DPP_SFM_COLMAP 1          /* path = the sparse model folder (.txt, or else .bin) */
#define L3DPP_SFM_MAVMAP 2          /* path = the result file */
#define L3DPP_SFM_OPENMVG 3         /* path = sfm_data.json */
#define L3DPP_SFM_PIX4D 4           /* path = the params folder, aux = the project prefix; the tie points are triangulated on CUDA device 0 */
#define L3DPP_SFM_COLMAP_LENSES 5   /* L3DPP_SFM_COLMAP with every camera's lens (l3dpp_sfm_lens) */
/* reads a model of one of the kinds above; NULL with the message in err for a malformed model or an unknown kind */
void* l3dpp_sfm_open(int kind, const char* path, const char* aux, char* err, int errcap);
void l3dpp_sfm_close(void* h);
int l3dpp_sfm_num_cameras(void* h);
/* camera i: head5 = id, has_K, focal, median depth, world point count; dist5 = radial[3], tangential[2]; -1 when i is out of range */
int l3dpp_sfm_camera(void* h, int i, double* head5, double* K9, double* R9, double* t3, double* C3, double* dist5, char* name, int namecap);
int l3dpp_sfm_worldpoints(void* h, int i, unsigned int* out, int cap);
/* lens of camera i as model, k[6], p[2] (9 doubles); -1 when i is out of range or the model was read without lenses */
int l3dpp_sfm_lens(void* h, int i, double* lens9);
void l3dpp_rotation_from_rpy(double roll, double pitch, double yaw, double* R9);
void l3dpp_decompose_projection(const double* P12, double* K9, double* R9, double* t3);
int l3dpp_sequential_neighbors(unsigned int i, unsigned int n_cams, unsigned int num_neighbors, unsigned int* out, int cap);

/* ---- the reference's binary files (csrc/line3d_bin.cc); no GPU is involved */
void* l3dpp_bin_open(const char* path, char* err, int errcap);
void l3dpp_bin_close(void* h);
void l3dpp_bin_sizes(void* h, long long* nlines, long long* nsegs, long long* nres);
/* arrays sized by l3dpp_bin_sizes: lines[nlines], clusters[nlines] (the cluster's line), segs[nsegs], res[nres] */
void l3dpp_bin_get(void* h, l3dpp_bin_line* lines, l3dpp_bin_seg* clusters, l3dpp_bin_seg* segs, l3dpp_bin_res* res);
/* the inverse of l3dpp_bin_get: lines[i].nseg / nres consecutive entries of segs / res belong to line i (their `line` field is not read) */
int l3dpp_bin_write(const char* path, long long nlines, const l3dpp_bin_line* lines, const l3dpp_bin_seg* clusters, const l3dpp_bin_seg* segs,
                    const l3dpp_bin_res* res, char* err, int errcap);
void* l3dpp_segcache_open(const char* path, char* err, int errcap);
void l3dpp_segcache_close(void* h);
long long l3dpp_segcache_count(void* h);
void l3dpp_segcache_get(void* h, float* xy4);
int l3dpp_segcache_write(const char* path, const float* xy4, long long n, char* err, int errcap);
/* segmentCachePath into buf; returns its length, or -1 if it does not fit */
int l3dpp_segcache_path(const char* folder, unsigned int cam, int w, int h, int max_img_width, char* buf, int cap);

#ifdef __cplusplus
}
#endif
#endif /* L3DPP_CAPI_H_ */
