/* include/l3d_capi.h — C ABI of libl3d_b200.so, the H100-native (sm_90a) replacement of Line3D++'s accelerator boundary.
 *
 * What it replaces (reference paths relative to manhofer/Line3Dpp):
 *   cudawrapper.h:54-80   match_lines_GPU / score_matches_GPU / replicator_dynamics_diffusion_GPU
 *   called from           line3D.cc:1060 (matchingGPU), line3D.cc:1365 (scoringGPU), line3D.cc:2033 (performRDD)
 * plus the host work the reference wraps around those calls and that this library moves onto the device:
 *   cudawrapper.cu:592-650 (dense D2H + host kNN pass), line3D.cc:811-858 (orientation check),
 *   line3D.cc:1311-1355 (sort + ranges + regularizers_tgt), line3D.cc:1672-1699 (inverse matches),
 *   line3D.cc:1586-1669 (filter + best estimate), line3D.cc:1852-1979 (affinity matrix), sparsematrix.cc:8-135.
 *
 * Conventions: plain pointers and sizes only; the caller owns every host buffer, the library owns every device
 * buffer; no ownership passes through the ABI (unlike SparseMatrix*& in cudawrapper.h:80).  Every entry returns
 * 0 on success or a negative l3d_status; l3d_last_error() gives the message (the reference prints CUDA errors to
 * cerr and carries on, dataArray.h:198-237).  A call that fails leaves its stage (views, matches, score sweep,
 * collinear lists, affinity matrix), and every stage computed from it, without a result: later calls that need one
 * return L3D_ERR_STATE.  The image calls (l3d_undistort_u8, l3d_undistort_map, l3d_remap_u8, l3d_undistort_points, l3d_prepare_gray_u8, l3d_decode_jpeg_gray_u8, l3d_decode_png_gray_u8) and the tie-point calls
 * (l3d_triangulate_points, l3d_median_depths) are not part of that chain: whether
 * they succeed or fail, every stage and its result stay as they were.  A context is single-owner (not thread-safe), one per GPU, and runs
 * on its own non-default stream.  There is NO CPU fallback: without a usable CUDA device l3d_ctx_create fails.
 */
#ifndef L3D_CAPI_H_
#define L3D_CAPI_H_
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

typedef struct l3d_ctx l3d_ctx;

typedef enum {
    L3D_OK = 0,
    L3D_ERR_INVALID = -1,      /* bad argument */
    L3D_ERR_CUDA = -2,         /* CUDA runtime error; see l3d_last_error */
    L3D_ERR_STATE = -3,        /* call order violated (e.g. match before set_views) */
    L3D_ERR_UNSUPPORTED = -4,  /* valid in the reference but not implemented here (yet) */
    L3D_ERR_NOMEM = -5
} l3d_status;

/* One view as the reference's View holds it after View::View (view.cc:6-42). */
typedef struct {
    uint32_t cam_id;        /* reference camID (line3D.h:104) */
    int32_t width, height;  /* image size */
    int32_t nseg;           /* number of 2D segments */
    float RtKinv[9];        /* (float) R^T K^-1, row-major          view.cc:37-40 (RtKinv_DA_) */
    float C[3];             /* (float) camera centre, UNtranslated  view.cc:35   (C_f3_)      */
    double RtKinv_d[9];     /* double R^T K^-1                      view.cc:27                */
    double C_d[3];          /* double camera centre in the (translated) working frame  view.cc:28, 510-514 */
    float k;                /* spatial regulariser k_               view.cc:301-314           */
    float median_depth;     /* median_depth_ (0 before matching)    view.h:108-121            */
} l3d_view_desc;

/* One emitted match of a source segment: the payload of L3DPP::Match (commons.h:186-203) minus the ids implied
 * by its position.  24 bytes. */
typedef struct {
    uint32_t tgt_seg;
    float overlap;
    float d_p1, d_p2, d_q1, d_q2;
} l3d_match_rec;

/* Full L3DPP::Match mirror (40 bytes), used by the pipeline dumps. */
typedef struct {
    uint32_t src_cam, src_seg, tgt_cam, tgt_seg;
    float overlap, score3D, d_p1, d_p2, d_q1, d_q2;
} l3d_match;

/* ---- context ------------------------------------------------------------------------------------------------ */
int l3d_ctx_create(int device, l3d_ctx** out);
void l3d_ctx_destroy(l3d_ctx* ctx);
const char* l3d_last_error(const l3d_ctx* ctx);
/* the CUDA stream the context launches on (cudaStream_t as void*), for event timing by the caller */
void* l3d_stream(l3d_ctx* ctx);
int l3d_sync(l3d_ctx* ctx);
/* number of kernels this context has launched so far (bench.py's gpu_launches) */
long long l3d_launch_count(const l3d_ctx* ctx);

/* ---- views: replaces initSrcDataGPU / per-pair uploads (line3D.cc:1018-1026, 1049-1057) ---------------------- */
/* segs_host[v] points to nseg*4 floats (x1,y1,x2,y2).  Data is device-resident after the call; a per-segment
 * pre-pass caches rays and plane normals (the reference recomputes them per pair, cudawrapper.cu:148-154). */
int l3d_set_views(l3d_ctx* ctx, int num_views, const l3d_view_desc* views, const float* const* segs_host);
/* same, all segments in ONE flat array (view v starts at the prefix sum of nseg); on_device != 0: the array is already
 * on this GPU (e.g. the output of the NCCL all-gather of per-view segment lists) and is used in place, not copied. */
int l3d_set_views_flat(l3d_ctx* ctx, int num_views, const l3d_view_desc* views, const float* segs_flat, int on_device);
/* update per-view k / median depth / double camera blocks without touching segments (after translate(), filter) */
int l3d_update_view_params(l3d_ctx* ctx, int num_views, const l3d_view_desc* views);

/* ---- matching: replaces match_lines_GPU (cudawrapper.h:54-64) for a whole batch of view pairs ----------------
 * pairs[2*i], pairs[2*i+1] = (src view index, tgt view index) into the l3d_set_views array;
 * F[9*i..] = float fundamental matrix of pair i, row-major, (float)F_double like eigen2dataArray line3D.cc:2775.
 * For every src segment the kNN tgt segments with the highest epipolar overlap among those with
 * overlap > epi_overlap and all four depths > 0 are kept (cudawrapper.cu:605-645); ties: smaller tgt_seg first.
 * 1 <= knn <= 32: the kNN best per src segment.  knn <= 0: keep ALL matches like the reference does (cudawrapper.cu:628-636),
 * in ascending tgt_seg order; the record array then uses the row stride l3d_match_stride() = the largest row of the job
 * (memory: total_rows * stride * 24 B).  knn > 32: the keep-all passes, then every row is cut to its knn best.
 * knn <= 0 and knn > 32: a row may hold at most 8533 matches before the cut (k_sort_rows sorts one row per warp in at most 200 KiB
 * of shared memory, 24 B per record); a longer row fails the call with L3D_ERR_UNSUPPORTED and leaves no match result.
 * Every call first builds the level-1 tables of its pairs (DESIGN.md section 2: the target segments of a pair as arcs of the
 * epipolar pencil, sorted): 16 B per (pair, target segment) kept until the next call + 28 B while they are built.
 * Results stay on the device; fetch with the l3d_get_* calls. */
int l3d_match_pairs(l3d_ctx* ctx, int num_pairs, const int32_t* pairs, const float* F, float epi_overlap, int knn);
/* sharded form (SURVEY.md 8e: view pairs are independent given all segment lists): the whole pair list is staged, so
 * row offsets and buffer sizes are those of the full job, but only pairs [first_pair, last_pair) are evaluated here;
 * the rows of the other pairs are filled in by the caller (l3d_match_device_buffers + a broadcast from their owner)
 * before l3d_score_sweep; for kNN <= 0 or > 32 the counts first, then l3d_match_restride(ctx, 0), then the records at that stride.
 * l3d_match_pairs == the range [0, num_pairs). */
int l3d_match_pairs_range(l3d_ctx* ctx, int num_pairs, const int32_t* pairs, const float* F, float epi_overlap, int knn,
                          int first_pair, int last_pair);
/* l3d_match_pairs + download in ONE call, overlapped (the shape of match_lines_GPU, which returns host lists): the pair
 * list is evaluated in `chunks` launches (1..64) and the counts / fixed-slot records of every finished chunk are copied to the
 * HOST arrays counts_out[total_rows], recs_out[total_rows*knn] on a second stream while the next chunk computes (page-locked
 * host memory needed for real overlap).  Asynchronous like the rest: l3d_sync() before reading.  1 <= knn <= 32. */
int l3d_match_pairs_host(l3d_ctx* ctx, int num_pairs, const int32_t* pairs, const float* F, float epi_overlap, int knn,
                         int32_t* counts_out, l3d_match_rec* recs_out, int chunks);
/* REF_CPU semantics (the reference built without CUDA or constructed with use_GPU=false, line3D.cc:49-53): matchingCPU's
 * double-precision twin of the path (line3D.cc:900-1015: mutualOverlap 1086-1165, triangulationDepths 1168-1193, depths
 * must exceed 1e-12) on the GPU.  Fd[9*i..] = the DOUBLE fundamental matrix of pair i.  Same outputs and accessors as
 * l3d_match_pairs_range; the scoring sweep that follows uses scoringCPU's rules (true per-camera maximum, line3D.cc:1208-1294)
 * and keeps the match lists in the reference's unsorted list order.  There is still no CPU fallback. */
int l3d_match_pairs_f64(l3d_ctx* ctx, int num_pairs, const int32_t* pairs, const double* Fd, float epi_overlap, int knn,
                        int first_pair, int last_pair);
/* Caller-given candidates: pair i with restricted[i] != 0 is matched only against its listed (source segment, target segment) cells;
 * the other pairs are scanned as l3d_match_pairs_range scans them.  triples[3*k..3*k+2] = (pair index, src_seg, tgt_seg), n of them, in
 * any order, duplicates allowed; src_seg indexes the pair's source view (pairs[2*i]), tgt_seg its target view.  A triple of a pair that
 * is not restricted, or not in [first_pair, last_pair), is checked and otherwise ignored; a restricted pair without triples has no
 * matches.  on_device != 0: triples is a device address on this GPU (restricted is always host memory); the call reads it on the
 * context's stream (l3d_stream), so work the caller queued there to fill it comes first, and work on other streams must be complete
 * (or made to precede with an event) before the call. */
typedef struct {
    const int32_t* restricted;      /* num_pairs flags */
    const int32_t* triples;         /* 3 * n */
    long long n;
    int32_t on_device;
} l3d_match_cand_desc;
/* l3d_match_pairs_range / l3d_match_pairs_f64 with candidates (DESIGN.md section 6c).  A row of a restricted pair keeps what the scan
 * would keep if its other target segments did not exist: the same exact arithmetic of the semantics, overlap > epi_overlap, the four
 * depth tests, kNN rule and tie order.  The outputs are those of the plain calls (counts, records, stride, l3d_match_total_matches,
 * l3d_match_gather, l3d_match_restride, l3d_score_sweep), except l3d_match_pair_evals: Ns*Nt for a scanned pair, the distinct triples
 * for a restricted one.  With every flag 0 the result is byte for byte the plain call's.  Rejected with L3D_ERR_INVALID before anything
 * is launched: a null descriptor or array, n < 0, a pair index outside [0, num_pairs), a src_seg outside [0, Ns) or a tgt_seg outside
 * [0, Nt) (l3d_last_error names the first such triple).  Waits for the device once, for the number of distinct triples; on_device also
 * reads the triples back to check them (3 * n * 4 bytes to the host) and waits for that. */
int l3d_match_pairs_cand(l3d_ctx* ctx, int num_pairs, const int32_t* pairs, const float* F, float epi_overlap, int knn, int first_pair,
                         int last_pair, const l3d_match_cand_desc* cand);
int l3d_match_pairs_cand_f64(l3d_ctx* ctx, int num_pairs, const int32_t* pairs, const double* Fd, float epi_overlap, int knn, int first_pair,
                             int last_pair, const l3d_match_cand_desc* cand);
/* slots per row of the record array of the last match result: knn, or the largest row when knn <= 0 was asked for */
int l3d_match_stride(const l3d_ctx* ctx);
#define L3D_SEM_REF_GPU 0
#define L3D_SEM_REF_CPU 1
/* semantics of the last match result (L3D_SEM_*), or < 0 */
int l3d_match_semantics(const l3d_ctx* ctx);
/* device addresses of the last match result: counts int32[total_rows], recs l3d_match_rec[total_rows*knn] (fixed slots) */
int l3d_match_device_buffers(l3d_ctx* ctx, void** counts_dev, void** recs_dev);
/* what the window scan of the matching kernel starts from for pair `pair`, one of the pairs the context's own last match call evaluated
 * (DESIGN.md section 2): windows_out[Ns * 20], per source row the pencil parameters k1, k2 of its two epipolar lines, 1 if the row
 * skips level 1, 0, then for every arc class c < 8 the first entry of the pair's sorted table inside class c whose arc start is not below
 * ka - 2^(21 + c) and the first whose start is above kb (pair-relative, over the whole class); basis_out[6] the pencil basis u, v;
 * class_off_out[10] the first sorted entry of every class and the end; arc_starts_out[Nt] the arc start of every sorted entry.  NULL
 * skips an output; a pair whose target view has no segments writes none; a pair restricted to caller-given candidates
 * (l3d_match_pairs_cand) has no table or windows and is rejected with L3D_ERR_INVALID. */
int l3d_match_row_windows(l3d_ctx* ctx, int pair, uint32_t* windows_out, double* basis_out, int32_t* class_off_out, uint32_t* arc_starts_out);
/* row_off_out[num_pairs+1]: first row of every pair in those buffers (prefix sum of Ns), last = total_rows */
int l3d_pair_row_offsets(l3d_ctx* ctx, long long* row_off_out);
/* pure host helper: contiguous split of n items with the given costs into `parts` ranges of near-equal cost;
 * bounds_out[parts+1], bounds_out[0] = 0, bounds_out[parts] = n. The same split on every rank. */
int l3d_balanced_split(const long long* cost, int n, int parts, int32_t* bounds_out);
/* in-process multi-GPU form of the sharded path: gather the rows of contexts that each matched a range of the same pair list into
 * dst.  Source i (src[i], any device, dst itself allowed) must hold the result of l3d_match_pairs_range / l3d_match_pairs_f64 over
 * exactly [pair_bounds[i], pair_bounds[i+1]) of the pair list dst matched: the same pairs, matrices, views, semantics, epi_overlap and
 * kNN.  pair_bounds[n_src+1] is non-decreasing within [0, num_pairs].  Afterwards dst holds what ONE such call over [pair_bounds[0],
 * pair_bounds[n_src]) would have left (the whole job for 0 and num_pairs): the same counts (0 outside that range), the same records up
 * to each row's count, the same l3d_match_stride, l3d_match_pair_evals and l3d_match_total_matches.
 *   1 <= kNN <= 32: the stride is kNN everywhere and rows are copied as they are.  kNN <= 0 or > 32: every source's stride is its own
 *   longest row; the gathered stride is the largest of them (what one context computes), dst re-lays its own rows if it has to, and
 *   the sources' rows are copied pitched (no kernel).
 * Asynchronous: dst's stream waits on an event recorded on every source's stream, so no host synchronisation is needed before the
 * call; the copies run on dst's stream.  The sources' buffers must stay alive and unchanged (no destroy, no new match call on them)
 * until dst's stream has passed the copies (l3d_sync(dst)).  Peer access to the sources' devices is enabled where the hardware allows
 * it (process-local runtime state); otherwise the runtime stages the copies.  Sources on dst's own device are plain device copies.
 * Errors: L3D_ERR_STATE for a dst or source without a match result, L3D_ERR_INVALID for another pair list or bounds that do not
 * match what the sources evaluated.  Failed or not, dst's scoring sweep and everything after it are dropped; a failed call also
 * drops dst's match result. */
int l3d_match_gather(l3d_ctx* dst, int n_src, l3d_ctx* const* src, const int32_t* pair_bounds);
/* re-lay the record array of the current match result at `stride` slots per row, wider or narrower; the counts and every row's records
 * up to its count stay as they are.  stride <= 0: the largest entry of the current count array (at least 1), reduced on the device.
 * This is how ranks that matched disjoint shares of a keep-all (kNN <= 0) or kNN > 32 job agree on one stride without another
 * collective: exchange the counts, call this with 0 (every rank now reduces the same counts), then exchange the records at the stride it
 * returns.  Returns the stride chosen, or L3D_ERR_STATE without a match result, L3D_ERR_INVALID for a stride below some row's count or
 * total_rows * stride >= 2^31 (the scoring sweep indexes slots in 32 bits).  Waits for the copy.  The buffer l3d_match_device_buffers
 * returned before is freed: ask again.  Failed or not, the scoring sweep and everything after it are dropped; a failed call also drops
 * the match result. */
int l3d_match_restride(l3d_ctx* ctx, int stride);
/* sizes of the last l3d_match_pairs result */
long long l3d_match_total_rows(const l3d_ctx* ctx);      /* sum of Ns over pairs */
long long l3d_match_total_matches(l3d_ctx* ctx);         /* matches of the last result (sum of the row counts), reduced on the device */
long long l3d_match_pair_evals(const l3d_ctx* ctx);      /* sum of Ns*Nt over pairs (distinct candidates of a restricted pair) */
/* counts_out[row_off(pair)+r] for all pairs (row_off = prefix sum of Ns in pair order); returns total matches */
long long l3d_get_match_counts(l3d_ctx* ctx, int32_t* counts_out);
/* one pair: counts_out[Ns], recs_out[Ns*knn] (slot r*knn+i valid for i < counts_out[r]) */
int l3d_get_pair_matches(l3d_ctx* ctx, int pair, int32_t* counts_out, l3d_match_rec* recs_out);
/* everything, compacted on the device to CSR before the D2H: row_ptr_out[total_rows+1], recs_out[capacity].
 * Returns the number of records (even if > capacity; then nothing is copied). */
long long l3d_get_matches_csr(l3d_ctx* ctx, int64_t* row_ptr_out, l3d_match_rec* recs_out, long long capacity);

/* ---- dense device contract of K_match_lines (cudawrapper.cu:186-253): one launch fills
 * depths[Ns*Nt] (float4: d_p1,d_p2,d_q1,d_q2 or -1) and overlaps[Ns*Nt], row-major by src.  Output pointers are
 * DEVICE pointers if out_on_device != 0, else host buffers.  HBM-write-bound: 20 B per pair evaluation. */
int l3d_match_dense(l3d_ctx* ctx, int src_view, int tgt_view, const float* F, float epi_overlap, float* depths,
                    float* overlaps, int out_on_device);

/* the same contract for many view pairs in ONE launch (tiles of all pairs in one grid).  pairs: (src, tgt) view indices, F: 9 floats per
 * pair, depths_dev[i] / overlaps_dev[i]: DEVICE pointers to pair i's Ns*Nt float4 / float outputs.  Asynchronous on the context's stream. */
int l3d_match_dense_pairs(l3d_ctx* ctx, int num_pairs, const int32_t* pairs, const float* F, float epi_overlap, float* const* depths_dev,
                          float* const* overlaps_dev);

/* test hook: same contract with the conservative pre-filter disabled (every cell through the exact path) */
int l3d_match_dense_nofilter(l3d_ctx* ctx, int src_view, int tgt_view, const float* F, float epi_overlap, float* depths,
                             float* overlaps, int out_on_device);

/* ---- scoring sweep: replaces, for ALL views in one call, the per-view sequence of Line3D::computeMatches after
 * matching (line3D.cc:745-773): checkMatchOrientation (811-858), scoringGPU incl. its host staging (1297-1414) and
 * score_matches_GPU (cudawrapper.h:67-74), storeInverseMatches (1672-1699), filterMatches (1586-1669).
 * Views are processed in ascending cam_id (the reference's std::map order); REF_GPU semantics (cudawrapper.cu:256-367).
 * Uses views[].k and views[].C_d / RtKinv_d of the last l3d_set_views / l3d_update_view_params call.
 *   two_sigA_sqr      2*sigma_a^2                          (line3D.cc:397)
 *   min_similarity    L3D_DEF_MIN_SIMILARITY_3D   0.50     (commons.h:58)
 *   min_best_score    L3D_DEF_MIN_BEST_SCORE_3D   0.75     (commons.h:59)
 *   min_best_perc     L3D_DEF_MIN_BEST_SCORE_PERC 0.10     (commons.h:60) */
int l3d_score_sweep(l3d_ctx* ctx, float two_sigA_sqr, float min_similarity, float min_best_score, float min_best_perc);
/* matches of one view after scoring in the reference's list order (segment; tgt cam; tgt seg).  kept_only != 0: only
 * those that survived filterMatches.  Returns the count (even if > cap). */
long long l3d_get_view_matches(l3d_ctx* ctx, int view, int kept_only, l3d_match* out, long long cap);
/* estimated_position3D_ (line3D.cc:1635-1647) in (view, segment) order: best match + unprojected P1,P2 (6 doubles, in
 * the working frame of C_d).  Returns the count. */
long long l3d_get_estimates(l3d_ctx* ctx, l3d_match* best_out, double* p1p2_out, long long cap);

/* ---- collinear 2D segments (optional, reconstruct3Dlines' collinearity_t > 0): replaces find_collinear_segments_GPU
 * (cudawrapper.h:76-78, K_collinearity cudawrapper.cu:370-429) called from View::findCollinGPU (view.cc:187) and the
 * host scan of its dense N x N char matrix (view.cc:192-203), for ALL views in one call.  Two segments of a view are
 * potentially collinear when neither endpoint of one projects onto the other and the larger of the mutual endpoint-to-
 * line distances is < dist_t pixels.  semantics: L3D_SEM_REF_GPU = the float kernel, L3D_SEM_REF_CPU = View::findCollinCPU
 * (view.cc:212-263, double geometry).  The result (View::collin_, ascending ids per segment) stays on the device: while it
 * is valid, l3d_affinity_matrix / l3d_affinity_edges add the collinearity links of computingAffinityMatrix
 * (line3D.cc:1904-1937, 1941-1974).  dist_t <= 1e-12 switches the links off again (line3D.cc:1752, 1905). */
int l3d_find_collinear(l3d_ctx* ctx, float dist_t, int semantics);
/* total number of list entries over all views (0 if off) */
long long l3d_collinear_total(const l3d_ctx* ctx);
/* collin_ of one view as CSR: row_ptr_out[nseg+1] relative to the view, idx_out[row_ptr_out[nseg]] segment ids.
 * Returns the view's entry count (even if > cap; then idx_out is not written). */
long long l3d_get_collinear(l3d_ctx* ctx, int view, long long* row_ptr_out, int32_t* idx_out, long long cap);

/* ---- affinity: Line3D::similarity (line3D.cc:1467-1553) for every kept match whose two segments have a 3D estimate,
 * i.e. the arithmetic of computingAffinityMatrix (line3D.cc:1852-1979).  Emits, in the reference's emission order,
 * the candidates with similarity > min_affinity (L3D_DEF_MIN_AFFINITY 0.5) as (global seg i, global seg j, w); the
 * "unused" de-duplication and local-id assignment stay on the host (line3D.cc:1881-1900, 1982-2023).  Needs
 * views[].median_depth to be current (l3d_update_view_params).  Returns the number of edges (even if > cap).
 * With collinearity links on (l3d_find_collinear) the list also holds the collinear candidates, each of which only
 * counts if its parent edge passed unused(): use l3d_affinity_matrix, which resolves that on the device.
 * min_affinity must be >= 0 (the reference's constant is 0.5): a segment without an estimate has similarity 0, and below 0 the
 * reference's loop would accept it, which the device does not model.  A negative or NaN min_affinity is rejected with
 * L3D_ERR_INVALID by this call and by l3d_affinity_matrix, and the rejected call drops any affinity matrix the context held. */
long long l3d_affinity_edges(l3d_ctx* ctx, float two_sigA_sqr, float med_scene_depth_lines, float min_affinity,
                             long long* out_gi, long long* out_gj, float* out_w, long long cap);

/* The complete affinity matrix on the device: the candidates of l3d_affinity_edges, then the reference's "unused" pair
 * filter (line3D.cc:1982-2002: only the first candidate of an unordered segment pair, in emission order) and first-come
 * local ids (line3D.cc:2005-2023), reproduced with stable sorts and atomic minima instead of mutex-protected maps; with
 * collinearity links the order-dependent "only if the parent edge was new" rule is resolved by a device fixpoint.
 * out_i/out_j/out_w: the CLEdge list A_ in the reference's order ((id1,id2,w),(id2,id1,w) per accepted edge);
 * out_local2global[id] = global segment index.  Returns the number of list entries (even if the capacities are too
 * small; then nothing is copied) and sets *num_ids. */
long long l3d_affinity_matrix(l3d_ctx* ctx, float two_sigA_sqr, float med_scene_depth_lines, float min_affinity, int* out_i,
                              int* out_j, float* out_w, long long cap_edges, long long* out_local2global, long long cap_ids,
                              long long* num_ids);

/* ---- diffusion: replaces replicator_dynamics_diffusion_GPU (cudawrapper.h:80, cudawrapper.cu:708-766) incl. the
 * SparseMatrix construction it needs (sparsematrix.cc:8-135).  Input: the CLEdge list A_ (clustering.h:47-51) as three
 * arrays and the number of rows n; iters = L3D_DEF_RDD_MAX_ITER (10).  Output: the diffused matrix as row-sorted COO
 * with nnz entries (what the reference downloads from W, line3D.cc:2036-2044).  No ownership transfer.
 * Ids are 0..n-1; an id without entries is allowed.  Each (i, j) may occur once: two equal entries would write one transposed
 * slot, a race in the reference too.  Weights must be finite and non-negative. */
int l3d_rdd(l3d_ctx* ctx, int n, long long nnz, const int* ei, const int* ej, const float* ew, int iters, int* out_i,
            int* out_j, float* out_w, float* kernel_ms);
/* performRDD (line3D.cc:2026-2076) on the affinity matrix that l3d_affinity_matrix left on the device: diffusion + the
 * min(w12, w21) symmetrisation without a host round trip; out_*: 2*K entries in (i, j) order.  Returns the entry count. */
long long l3d_rdd_affinity(l3d_ctx* ctx, int iters, int32_t* out_i, int32_t* out_j, float* out_w, long long cap);

/* ---- line bundling (optional, reconstruct3Dlines' use_CERES): replaces LineOptimizer::optimize (optimization.h:174-190,
 * optimization.cc:8-303; called from Line3D::optimizeClusters line3D.cc:2269-2275), i.e. the Ceres problem the reference
 * builds from LineReprojectionError (optimization.h:52-171) with every camera / intrinsic block constant.  Only the four
 * Cayley parameters of each line are free, so the system is block diagonal: residuals, exact derivatives, the 4x4
 * Levenberg-Marquardt solves and the candidate costs run on the device for all lines at once; the host plays Ceres'
 * trust-region controller (one radius, its default tolerances).  Ceres itself is not needed.
 *   p1p2        6 doubles per line: the cluster's 3D segment in the working (translated) frame   optimization.cc:36-39
 *   res_ptr     num_lines+1 offsets into the residual arrays: res_ptr[0] == 0 and non-decreasing (else L3D_ERR_INVALID,
 *               checked before anything is uploaded); line i owns residuals res_ptr[i] .. res_ptr[i+1]-1
 *   res_cam     per residual: index into cams
 *   res_xy      per residual: x1 y1 x2 y2 of the observed 2D segment (View::getLineSegment2D)     optimization.cc:155-166
 *   cams        16 doubles per camera: R (row-major), C (working frame), fx, fy, px, py           optimization.cc:108-141
 *   max_iter    L3D_DEF_CERES_MAX_ITER 250 (commons.h:88)
 *   p1p2_out    updated segments (unit direction around the old mid point, optimization.cc:259-277); may alias p1p2
 *   valid_out   0 where the reference drops the cluster (optimization.cc:293-298)
 *   summary     optional, 8 doubles: iterations, initial cost, final cost, termination (0 convergence, 1 max_iter reached,
 *               2 failure), successful steps, free lines, final trust-region radius, kernels launched.  Both costs are 0
 *               when the first evaluation fails (a residual block with omega or the projected line's norm below 1e-12). */
int l3d_optimize_lines(l3d_ctx* ctx, int num_lines, const double* p1p2, const long long* res_ptr, const int32_t* res_cam,
                       const double* res_xy, int num_cams, const double* cams, int max_iter, double* p1p2_out, int32_t* valid_out,
                       double* summary);

#define L3D_LENS_RADTAN 0       /* OpenCV's standard model: k1 k2 p1 p2 k3 [k4 k5 k6] */
#define L3D_LENS_FISHEYE 1      /* OpenCV's fisheye (equidistant) model: k1..k4 */
/* ---- lens undistortion of 8-bit images: Line3D::undistortImage (line3D.cc:83-109), i.e. OpenCV's initUndistortRectifyMap with
 * fixed-point maps (CV_16SC2 pixel + CV_16UC1 1/32-px fraction) followed by remap(INTER_LINEAR, BORDER_CONSTANT 0), output the size
 * and type of the input, K unchanged.  The camera matrix is [[fx,0,cx],[0,fy,cy],[0,0,1]] (skew is ignored, as in the reference);
 * the distortion vector is (k1, k2, p1, p2, k3, k4, k5, k6) = (radial[0], radial[1], tangential[0], tangential[1], radial[2],
 * rational[0..2]).  model = L3D_LENS_FISHEYE instead is cv::fisheye::initUndistortRectifyMap(K, fisheye[0..3], I, K) with the same
 * fixed-point maps; radial, tangential and rational must then be zero.  The maps are defined by the formulas of DESIGN.md §4a,
 * which OpenCV builds reproduce to within one 1/32-px step (radtan: exactly, for the rational terms too, up to OpenCV's accumulation
 * order; fisheye: up to the last ulp of atan); the remap is bit-exact to OpenCV's.  Pixels are interleaved (channels 1 or 3);
 * pitches are row strides in bytes.
 * Rejected with L3D_ERR_INVALID: width or height outside [1, 32767], channels other than 1 or 3, a pitch below width*channels,
 * null pointers, src == dst, fx or fy zero or not finite, a principal point or coefficient that is not finite, an unknown model,
 * a fisheye descriptor with a nonzero radial, tangential or rational term.
 * on_device != 0: every pointer is a device address on this GPU and the call is asynchronous on the context's stream;
 * on_device == 0: host buffers, staged through the context's own device buffers, and the call returns when the output is written. */
typedef struct {
    int32_t width, height, channels;
    int64_t src_pitch, dst_pitch;
    const uint8_t* src;
    uint8_t* dst;
    double fx, fy, cx, cy;
    double radial[3], tangential[2];
    /* lens model; a zero-initialised tail is the model above (L3D_LENS_RADTAN without rational terms) */
    int32_t model;                 /* L3D_LENS_RADTAN or L3D_LENS_FISHEYE */
    double rational[3];            /* L3D_LENS_RADTAN: k4, k5, k6 (the denominator of OpenCV's 8-coefficient model) */
    double fisheye[4];             /* L3D_LENS_FISHEYE: k1..k4 of theta_d = theta (1 + k1 theta^2 + k2 theta^4 + k3 theta^6 + k4 theta^8) */
    /* OpenCV's newCameraMatrix and newImageSize; a zero-initialised tail is the camera's own K and the source size, as above.
     * With them the maps are initUndistortRectifyMap(K, D, I, newK, newSize) (fisheye: cv::fisheye's, with P = newK): the output
     * pixel (j, i) is taken back through inv(newK) (by cofactors, as above), distorted and projected with the camera's fx, fy, cx, cy.
     * The output is out_height x out_width: l3d_undistort_u8 writes that many rows to dst with dst_pitch >= out_width * channels;
     * l3d_undistort_map returns maps of that size; l3d_remap_u8 reads a width x height source with maps of the output size.
     * Rejected with L3D_ERR_INVALID: a new K that is not all zero and has new_fx or new_fy zero or not finite, or new_cx or new_cy
     * not finite; an output size other than (0, 0) with a value outside [1, 32767].  Skew is ignored here too.  DESIGN.md §4a. */
    double new_fx, new_fy, new_cx, new_cy;   /* all four 0: the camera's own K */
    int32_t out_width, out_height;           /* both 0: the source size */
} l3d_undistort_desc;
/* undistort n images in one launch; images, sizes, channel counts and cameras may all differ */
int l3d_undistort_u8(l3d_ctx* ctx, int n, const l3d_undistort_desc* descs, int on_device);
/* the fixed-point maps of one image (src, dst and the pitches are not used): map_xy int16[out_height*out_width*2] (x, y per pixel),
 * map_frac uint16[out_height*out_width] = (v & 31) * 32 + (u & 31); rows packed.  What cv::remap takes as its two maps. */
int l3d_undistort_map(l3d_ctx* ctx, const l3d_undistort_desc* desc, int16_t* map_xy, uint16_t* map_frac, int on_device);
/* cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) of one image with caller-given maps in that layout, of the output size (the camera and
 * the new K are not used) */
int l3d_remap_u8(l3d_ctx* ctx, const l3d_undistort_desc* desc, const int16_t* map_xy, const uint16_t* map_frac, int on_device);

/* ---- lens undistortion of points: OpenCV 4.13's cv::undistortPoints(src, dst, K, D, noArray(), P) for a RADTAN lens (its fixed five
 * iterations, the fallback to the undistorted-camera point when the distortion factor turns negative, the final cast to float) and
 * cv::fisheye::undistortPoints(src, dst, K, D, I, P) with its default criteria for a FISHEYE lens (at most ten Newton steps; a point that
 * does not converge or whose angle changes sign gives (-1e6, -1e6)), with P the new camera matrix of `cam` (all zero: K).  The output is
 * in pixels of P.  Points are float32 (x, y) pairs, e.g. the endpoints of segments (x1, y1, x2, y2); NaN and infinite inputs are computed
 * as OpenCV computes them.  RADTAN output is bit-identical to OpenCV's; FISHEYE output may differ where the device's tan differs from
 * the host's (DESIGN.md §4a).  dst == src is allowed; other overlaps between sets are not.  Only the camera, lens and new-K fields of
 * `cam` are read (width, height, channels, the image pointers, pitches and output size are ignored) and checked as l3d_undistort_u8
 * checks them, with the same messages; also rejected with L3D_ERR_INVALID: n < 0, a null descriptor array, count < 0, a null src or dst
 * when count > 0.  on_device as for l3d_undistort_u8 (src and dst are device addresses, or host arrays staged through the context's
 * buffers).  Not part of the pipeline chain: every stage and its result stay as they were. */
typedef struct {
    l3d_undistort_desc cam;        /* the camera, its lens and the new camera matrix */
    int64_t count;                 /* number of points */
    const float* src;              /* count (x, y) pairs */
    float* dst;                    /* count (x, y) pairs */
} l3d_points_desc;
/* undistort n point sets in one launch (one thread per point); cameras, lenses and lengths may all differ */
int l3d_undistort_points(l3d_ctx* ctx, int n, const l3d_points_desc* sets, int on_device);

/* ---- image preparation for line detection: what the reference's detectLineSegments (line3D.cc:249-289) does to an image before LSD
 * sees it.  cvtColor(CV_RGB2GRAY) for 3 channels (channel 0 is R; OpenCV's 15-bit fixed point) or the grey pixels as they are, then,
 * when max_img_width > 0 and the larger side exceeds it, cv::resize(gray, out, Size(), s, s) with INTER_LINEAR and
 * s = float(max_img_width) / float(max(width, height)); OpenCV turns a source step of exactly 2 into the 2x2 INTER_AREA mean.  Bit-exact
 * to OpenCV 4.13's x86 build (DESIGN.md §4b).  One fused kernel per call: no grey intermediate is stored.
 * out_width / out_height must be what l3d_image_prep_size returns for width, height and max_img_width (the caller sizes dst with it).
 * Rejected with L3D_ERR_INVALID: width or height outside [1, 32767], channels other than 1 or 3, out_width / out_height other than
 * l3d_image_prep_size's, a src pitch below width*channels or a dst pitch below out_width, null pointers, src == dst.
 * on_device as for l3d_undistort_u8.  Not part of the pipeline chain: every stage and its result stay as they were. */
typedef struct {
    int32_t width, height, channels;   /* source image; channels 1 or 3, interleaved */
    int32_t max_img_width;             /* the Line3D constructor's argument; <= 0: no resize */
    int64_t src_pitch, dst_pitch;      /* row strides in bytes */
    const uint8_t* src;
    uint8_t* dst;                      /* out_height rows of out_width grey bytes */
    int32_t out_width, out_height;     /* from l3d_image_prep_size */
} l3d_image_prep_desc;
/* the size of the prepared image (the rounding of the segment cache's file name, segmentCachePath); returns 1 if the image is resized,
 * 0 if not, L3D_ERR_INVALID for a size outside [1, 32767] or a null output pointer.  Needs no context and no GPU. */
int l3d_image_prep_size(int width, int height, int max_img_width, int32_t* out_width, int32_t* out_height);
/* prepare n images in one launch; sizes, channel counts and max_img_width may all differ */
int l3d_prepare_gray_u8(l3d_ctx* ctx, int n, const l3d_image_prep_desc* descs, int on_device);

/* ---- JPEG decoding: the first step of every frontend's image loop (main_vsfm.cpp:267-306 and its five siblings), cv::imread(path,
 * IMREAD_GRAYSCALE), byte for byte as OpenCV 4.13 returns it on x86: the Y component of a baseline or extended-sequential Huffman JPEG
 * (no colour conversion, no upsampling), libjpeg-turbo's accurate integer IDCT as its SIMD code computes it, then OpenCV's EXIF
 * orientation (1..8; any other value, a missing or a broken EXIF block: none).  DESIGN.md §4c.
 * Supported: SOF0 / SOF1 with 8-bit samples, 8- or 16-bit DQT, one component or three (YCbCr) with Y at the largest sampling factors,
 * interleaved and non-interleaved scans, restart intervals, APPn / COM / fill bytes.  Rejected with a message that names the reason:
 * progressive, lossless, hierarchical and arithmetic-coded files, 12-bit samples, DNL, 2 or 4 components, RGB (Adobe transform 0, or
 * component ids 'R' 'G' 'B' without JFIF), Y below the largest sampling factors, a side outside [1, 32767], a missing table, EOI or
 * component scan, and corrupt or truncated data (no attempt is made at libjpeg's recovery).
 * Not part of the pipeline chain: every stage and its result stay as they were. */
/* size of imread(IMREAD_GRAYSCALE)'s output (after EXIF orientation); needs no context and no GPU.  L3D_OK, or L3D_ERR_INVALID for a
 * file outside the subset above (readJPEGSize of include/line3d_io.h gives the reason) or a null pointer */
int l3d_jpeg_info(const uint8_t* data, int64_t size, int32_t* out_width, int32_t* out_height);
typedef struct {
    const uint8_t* data; int64_t size;   /* the file's bytes, always HOST memory (the headers are parsed on the host) */
    uint8_t* dst; int64_t dst_pitch;     /* out_height rows of out_width grey bytes */
    int32_t out_width, out_height;       /* from l3d_jpeg_info */
} l3d_jpeg_desc;
/* decode n files in two launches (Huffman decoding: one thread per entropy-coded segment; IDCT and store: one thread per 8x8 block);
 * sizes, sampling, restart intervals and orientations may all differ.  on_device != 0: dst (only) is a device address on this GPU;
 * on_device == 0: dst is host memory, staged through the context's own device buffers.  Either way only the coded bytes of Y's scan
 * are uploaded, and the call returns when its result is known: bytes of dst beyond each row's out_width stay untouched.
 * A descriptor with no data, a file outside the subset, a null dst, an out size other than l3d_jpeg_info's or a dst_pitch below
 * out_width is rejected (L3D_ERR_INVALID, l3d_last_error naming the first bad index and the reason) before anything is launched.
 * Corrupt entropy-coded data (no Huffman code matches, AC coefficients past index 63, a segment that ends early) is found on the GPU:
 * L3D_ERR_INVALID naming the first such image; host dst buffers are then untouched, device ones hold undefined bytes. */
int l3d_decode_jpeg_gray_u8(l3d_ctx* ctx, int n, const l3d_jpeg_desc* descs, int on_device);

/* ---- PNG decoding: cv::imread(path, IMREAD_GRAYSCALE) of a PNG file, byte for byte as OpenCV 4.13 returns it on x86 (libpng's
 * conversions as OpenCV sets them up, then OpenCV's EXIF orientation from an eXIf chunk).  DESIGN.md §4d.
 * Supported: every colour type and bit depth, Adam7 interlacing, PLTE (indices past its entries read black), tRNS (no effect: alpha
 * is dropped), gAMA / sRGB on grey images (no effect) and on colour images of 8 bits or less (libpng's gamma tables), eXIf, split and
 * empty IDAT chunks, ancillary chunks that do not change the pixels.  Rejected with a message that names the reason: a bad CRC in
 * any chunk, iCCP, cHRM, cICP, gamma on 16-bit colour, APNG chunks, chunks out of place, unknown critical chunks, a palette image
 * without PLTE, a side above 1,000,000 or more than 2^30 pixels, a bad zlib header or preset dictionary, and corrupt data that
 * libpng would only warn about (extra compressed data, data after the zlib stream) or fail on.
 * Not part of the pipeline chain: every stage and its result stay as they were. */
/* size of imread(IMREAD_GRAYSCALE)'s output (after EXIF orientation); needs no context and no GPU.  L3D_OK, or L3D_ERR_INVALID for a
 * file outside the subset above (readPNGSize of include/line3d_io.h gives the reason) or a null pointer */
int l3d_png_info(const uint8_t* data, int64_t size, int32_t* out_width, int32_t* out_height);
typedef struct {
    const uint8_t* data; int64_t size;   /* the file's bytes, always HOST memory (the chunks are parsed on the host) */
    uint8_t* dst; int64_t dst_pitch;     /* out_height rows of out_width grey bytes */
    int32_t out_width, out_height;       /* from l3d_png_info */
} l3d_png_desc;
/* decode n files in three launches (inflate: one warp per image; unfiltering: a diagonal wavefront over bands of rows per Adam7
 * pass; grey conversion and store: one thread per output pixel); sizes, formats and orientations may all differ.  on_device as for
 * l3d_decode_jpeg_gray_u8; only the IDAT payload is uploaded, and bytes of dst beyond each row's out_width stay untouched.
 * A descriptor with no data, a file outside the subset, a null dst, an out size other than l3d_png_info's or a dst_pitch below
 * out_width is rejected (L3D_ERR_INVALID, l3d_last_error naming the first bad index and the reason) before anything is launched.
 * A corrupt zlib stream (bad block type, stored length, code-length set or code, a distance past the output start or the window,
 * too much or too little data, data after the stream, a wrong Adler-32) or a bad filter type is found on the GPU: L3D_ERR_INVALID
 * naming the first such image; host dst buffers are then untouched, device ones hold undefined bytes. */
int l3d_decode_png_gray_u8(l3d_ctx* ctx, int n, const l3d_png_desc* descs, int on_device);

/* ---- tie-point triangulation:linearHomTriangulation of the reference's Pix4D frontend (main_pix4d.cpp:34-70, 354-372) for every point
 * in one launch.  Point i has the observations [obs_ptr[i], obs_ptr[i+1]) (obs_ptr[0] = 0): camera obs_cam[o] in [0, n_cams) and image
 * point (obs_xy[2o], obs_xy[2o+1]); P: the 3x4 projection matrix of every camera, 12 doubles row-major.  A point with fewer than three
 * observations is invalid with X = 0, as the reference skips it.  Otherwise A^T A (4x4, double) is accumulated from the rows Sx P[cam]
 * in observation order, its eigenvector v of the smallest eigenvalue is found by cyclic Jacobi in double, X = v.xyz / v.w, and
 * valid = |X| > L3D_EPS (1e-12) compared as the reference does: NaN is invalid, +-Inf is valid.  Not bit-exact to Eigen's JacobiSVD:
 * the contract is the tolerance of DESIGN.md §6b.  X_out: 3 doubles per point; valid_out: 0 / 1 per point.
 * on_device != 0: every pointer is a device address on this GPU and the call is asynchronous on the context's stream; an observation
 * of a camera outside [0, n_cams) then makes its point invalid.  on_device == 0: host arrays, checked (L3D_ERR_INVALID for a decreasing
 * obs_ptr or an unknown camera), staged through the context's own buffers; the call returns when the outputs are written. */
int l3d_triangulate_points(l3d_ctx* ctx, long long n_points, const int64_t* obs_ptr, const int32_t* obs_cam, const double* obs_xy, int n_cams,
                           const double* P, double* X_out, int32_t* valid_out, int on_device);
/* per-camera median depth of main_pix4d.cpp:386-418: camera c lists the points [list_ptr[c], list_ptr[c+1]) of list_pts (ids into X /
 * valid, repeats allowed); count_out[c] = the number of list entries whose point is valid, median_out[c] = the element at count/2 of
 * their float depths (float)|X - C[c]| sorted ascending, 0 when there are none.  One device pass: depths, a segmented sort, a pick;
 * exact given X.  At most 2^31 - 1 list entries per call.  on_device as for l3d_triangulate_points (a point id outside [0, n_points)
 * counts as invalid on the device and is rejected on the host). */
int l3d_median_depths(l3d_ctx* ctx, int n_cams, const int64_t* list_ptr, const int32_t* list_pts, long long n_points, const double* X,
                      const int32_t* valid, const double* C, int32_t* count_out, float* median_out, int on_device);

/* ---- visual neighbours from camera poses (DESIGN.md §6d): for models without world points (mavmap, SLAM or VIO keyframes, RTK-posed
 * surveys, SfM exports without structure).  Every view i gets gx * gy virtual world points, the pixel centres ((c + 0.5) width / gx,
 * (r + 0.5) height / gy) back-projected to camera depth median_depth (sample s = r * gx + c is point i * gx * gy + s).  A point is
 * observed by its own view and by every other view j that sees it in front (depth > 0) and inside [0, width) x [0, height), without
 * occlusion or depth-range tests; all of that in IEEE double in the operation order of DESIGN.md §6d.  n_i is the number of points
 * view i observes (its own included), common(i, j) the number both observe.  The neighbours are then find_visual_neighbors' (i.e.
 * findVisualNeighborsFromWPs', line3D.cc:578-699) for those points: score 2 common / (n_i + n_j) in float, optical axes under 1.571
 * rad, common > 4, the 0.8 cut, the distance resort and the greedy baseline > 0.1 loop, with camera centres, axes and distances
 * computed from K, R, t as addImage computes them (no translation is applied).  Not part of the pipeline chain: every stage and its
 * result stay as they were. */
typedef struct {
    uint32_t cam_id;                /* the camID the lists name; unique */
    int32_t width, height;          /* image size, at least 1 */
    int32_t pad;                    /* 0 */
    double fx, fy, cx, cy, skew;    /* K = [[fx, skew, cx], [0, fy, cy], [0, 0, 1]]; fx, fy nonzero */
    double R[9];                    /* row-major, x_cam = R X + t */
    double t[3];
    double median_depth;            /* depth of the virtual points in front of this view; finite, > 0 */
} l3d_pose_view;
#define L3D_POSE_MAX_VIEWS 50000             /* the co-visibility histogram of a view: 4 bytes per view in shared memory */
#define L3D_POSE_MAX_POINTS (1ll << 26)      /* the largest n * gx * gy (24 bytes of virtual point per sample on the device) */
/* The neighbours of n views as CSR: view i's are nb_cam[nb_ptr[i] .. nb_ptr[i+1]), camIDs in ascending order (the lists for addImage
 * with neighbors_by_worldpoints = false).  nb_ptr[n+1] is always written; nb_cam only when the total fits cap (n * min(num_neighbors,
 * n - 1) always does).  n_obs_out (n entries, or NULL): n_i.  timing_out (2 doubles, or NULL): the device time of the kernels in ms
 * (CUDA events) and the host time of the selection in ms.  Returns the total number of neighbour entries or a negative status.
 * Rejected with L3D_ERR_INVALID, l3d_last_error naming the view (index and camID): median_depth <= 0 or not finite, width or height
 * below 1, fx or fy zero or not finite, cx, cy or skew not finite, R or t not finite, a camID that repeats an earlier view's; and
 * gx or gy below 1, n < 0, a null views or nb_ptr array.  L3D_ERR_UNSUPPORTED: n above L3D_POSE_MAX_VIEWS, n * gx * gy above
 * L3D_POSE_MAX_POINTS, more than 2^31 - 1 observations (the sum over points of their observers) or co-visibility slots. */
long long l3d_pose_neighbors(l3d_ctx* ctx, int n, const l3d_pose_view* views, int gx, int gy, unsigned int num_neighbors, int64_t* nb_ptr,
                             uint32_t* nb_cam, long long cap, int32_t* n_obs_out, double* timing_out);
/* test export of the same device pass: n_obs_out (n entries, or NULL) and every nonzero (i, j, common(i, j)), i != j, as view
 * indices, ascending in (i, j), 3 int32 each in ijc_out when they fit cap triples.  Returns the number of triples or a negative
 * status; rejections as l3d_pose_neighbors'. */
long long l3d_pose_covisibility(l3d_ctx* ctx, int n, const l3d_pose_view* views, int gx, int gy, int32_t* n_obs_out, int32_t* ijc_out, long long cap);

/* stable ascending argsort of float keys on the device: the weight sort of performClustering (clustering.cc:13-14) for
 * large edge lists.  perm_out[i] = index of the i-th smallest key, ties in input order. */
int l3d_argsort_f32(l3d_ctx* ctx, long long n, const float* keys, unsigned int* perm_out);

/* measurement aid: achieved non-tensor FP32 FFMA throughput of this GPU right now (TFLOP/s), the denominator of the
 * fused kernel's compute roofline */
int l3d_fp32_peak_probe(l3d_ctx* ctx, double* tflops_out);

#ifdef __cplusplus
}
#endif
#endif /* L3D_CAPI_H_ */
