/* oracle/l3d_oracle.h — C ABI of the CPU ORACLE.  TEST INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load
 * liboracle.so.  The product library (line3dpp_b200/csrc) never includes, links or calls anything here.
 *
 * Parity status (see DESIGN.md "Oracle pinning"): PINNED.
 *   - kernel-level functions (orc_match_*_f32, orc_score_matches_f32, orc_rdd_f32, orc_cluster) against the reference's own
 *     cudawrapper.cu / sparsematrix.cc / clustering.cc compiled in place (oracle/_ref) and against golden vectors those produced
 *     on the GPU (tests/golden/ref_kernels_v1.npz, ref_collinear_v1.npz).
 *   - the restatement of the line3D.cc / view.cc host logic (the orc_ctx pipeline) against the reference's WHOLE pipeline compiled
 *     verbatim (oracle/ref_full_harness.cu -> oracle/_ref/libl3dref_full_{cpu,gpu}.so, Eigen/OpenCV/Boost replaced by the header
 *     stand-ins of oracle/ref_shim): index-exact at every stage on synthetic scenes (live) and on the vsfm_result.nvm inputs
 *     (tests/golden/ref_full_nvm_cpu_v1.npz), tests/test_ref_full_cpu.py.
 */
#ifndef L3D_ORACLE_H_
#define L3D_ORACLE_H_
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* flat mirror of L3DPP::Match (commons.h:186-203) — same layout as ref_match_t in ref_harness.cu */
typedef struct {
    uint32_t src_cam, src_seg, tgt_cam, tgt_seg;
    float overlap, score3D, d_p1, d_p2, d_q1, d_q2;
} orc_match_t;

/* one collinear 3D segment of a final line + the index of the line it belongs to */
typedef struct { int line; double p1[3], p2[3]; } orc_seg3d_t;
/* one 2D residual of a final line */
typedef struct { int line; uint32_t cam, seg; } orc_residual_t;

/* ---- kernel-level functions: same signatures as ref_harness.cu's ref_* so tests can swap them ---- */
int orc_match_dense_f32(const float* lines_src, int Ns, const float* lines_tgt, int Nt, const float* F,
                        const float* RtKinv_src, const float* RtKinv_tgt, const float* C_src, const float* C_tgt,
                        float epi_overlap, float* depths_out, float* overlaps_out, float* kernel_ms);
long long orc_match_lines_f32(const float* lines_src, int Ns, const float* lines_tgt, int Nt, const float* F,
                              const float* RtKinv_src, const float* RtKinv_tgt, const float* C_src,
                              const float* C_tgt, uint32_t srcCamID, uint32_t tgtCamID, float epi_overlap, int kNN,
                              int* counts, orc_match_t* out, int cap, double* wall_ms);
/* matchingCPU (line3D.cc:900-1015) on explicit double cameras: F, RtKinv_*, C_* are double here */
long long orc_match_lines_f64(const float* lines_src, int Ns, const float* lines_tgt, int Nt, const double* F,
                              const double* RtKinv_src, const double* RtKinv_tgt, const double* C_src,
                              const double* C_tgt, uint32_t srcCamID, uint32_t tgtCamID, float epi_overlap, int kNN,
                              int* counts, orc_match_t* out, int cap, double* wall_ms);
int orc_score_matches_f32(const float* lines, int Ns, const float* matches, int M, const int* ranges,
                          const float* reg_tgt, const float* RtKinv, const float* C, float two_sigA_sqr, float k,
                          float min_similarity, float* scores_out, float* kernel_ms);
int orc_rdd_f32(int nedges, const int* ei, const int* ej, const float* ew, int n, int* out_i, int* out_j,
                float* out_w, double* wall_ms);
/* the same with `iters` diffusion iterations instead of L3D_DEF_RDD_MAX_ITER (10) */
int orc_rdd_f32_iters(int nedges, const int* ei, const int* ej, const float* ew, int n, int iters, int* out_i, int* out_j,
                      float* out_w, double* wall_ms);
/* find_collinear_segments_GPU + K_collinearity (cudawrapper.cu:370-429, 689-705) / View::findCollinCPU (view.cc:212-263):
 * dense N x N char matrix C[r*N+c] = 1 iff segment c is collinear with segment r (distance threshold dist_t, px) */
int orc_collinear_f32(const float* lines, int N, float dist_t, unsigned char* C_out, float* kernel_ms);
int orc_collinear_f64(const float* lines, int N, float dist_t, unsigned char* C_out, float* kernel_ms);
int orc_cluster(int nedges, const int* ei, const int* ej, const float* ew, int n, float c, int* labels_out);

/* LineOptimizer::optimize (optimization.cc:8-303) + LineReprojectionError (optimization.h:52-171) with Ceres' published
 * Levenberg-Marquardt (Ceres itself is a third-party dependency absent from the reference tree).  cams: 16 doubles per
 * camera (R row-major, C, fx, fy, px, py); res_cam indexes cams; res_xy = x1 y1 x2 y2 per residual; valid_out 0 = dropped.
 * summary[8] (optional): iterations, initial cost, final cost, termination (0 conv, 1 max iter, 2 failure), successful steps,
 * free lines, final radius, 0. */
int orc_optimize_lines(int num_lines, const double* p1p2, const long long* res_ptr, const int* res_cam, const double* res_xy, int num_cams,
                       const double* cams, int max_iter, double* p1p2_out, int* valid_out, double* summary);

/* ---- pipeline: restatement of L3DPP::Line3D (line3D.h:80-233) ---- */
typedef struct orc_ctx orc_ctx;
/* use_gpu: 1 = REF_GPU semantics (float kernels, scoringGPU), 0 = REF_CPU (matchingCPU/scoringCPU)   line3D.cc:49-53 */
orc_ctx* orc_create(int neighbors_by_worldpoints, int use_gpu);
void orc_destroy(orc_ctx*);
/* optional: route the three accelerator calls through other implementations with the ref_* signatures
 * (e.g. the verbatim reference kernels from oracle/_ref on a GPU box).  NULL keeps the CPU emulation. */
void orc_set_backend(orc_ctx*, void* match_lines_fn, void* score_matches_fn, void* rdd_fn);
void orc_set_threads(int n);
/* same for find_collinear_segments_GPU (signature of ref_collinear / orc_collinear_f32); NULL restores the CPU emulation */
void orc_set_collinear_backend(orc_ctx*, void* collinear_fn);
/* optional: the match lists of every view pair from fn instead of from matching (matchingGPU / matchingCPU), so that hand-built
 * lists reach the orientation check, scoring and filter of either semantics.  fn(src cam, tgt cam, Ns, Nt, kNN, counts[Ns],
 * out[Ns * cap], cap) fills row r's counts[r] <= cap matches at out[r * cap] and returns their total.  NULL: matching again. */
typedef long long (*orc_match_source_fn)(uint32_t src_cam, uint32_t tgt_cam, int Ns, int Nt, int kNN, int* counts, orc_match_t* out, int cap);
void orc_set_match_source(orc_ctx*, orc_match_source_fn fn);
/* addImage with explicit line segments (line3D.cc:112-226); image itself is not needed */
int orc_add_view(orc_ctx*, uint32_t cam_id, int width, int height, const double* K, const double* R, const double* t,
                 float median_depth, const uint32_t* wps_or_neighbors, int n_list, const float* segs, int nseg);
int orc_match_images(orc_ctx*, float sigma_p, float sigma_a, uint32_t num_neighbors, float epi_overlap, int kNN,
                     float const_reg_depth);
int orc_reconstruct(orc_ctx*, uint32_t visibility_t, int perform_diffusion, float collinearity_t);
/* same with the bundling step of reconstruct3Dlines (use_CERES, max_iter_CERES; line3D.cc:1800-1805) */
int orc_reconstruct_opt(orc_ctx*, uint32_t visibility_t, int perform_diffusion, float collinearity_t, int use_ceres, uint32_t max_iter_ceres);
int orc_get_opt_summary(orc_ctx*, double* summary8);

/* stage dumps (all in deterministic single-thread reference order) */
int orc_num_views(orc_ctx*);
long long orc_pair_evals(orc_ctx*);                 /* sum of Ns*Nt over matched view pairs */
int orc_get_pairs(orc_ctx*, int* src_tgt, int cap); /* matched (src,tgt) cam pairs in match order; returns count */
long long orc_get_matches(orc_ctx*, uint32_t cam, orc_match_t* out, long long cap); /* surviving matches of a view */
long long orc_get_scored(orc_ctx*, uint32_t cam, orc_match_t* out, long long cap);  /* matches right after scoring */
int orc_get_view_info(orc_ctx*, uint32_t cam, float* k, float* median_depth);
long long orc_get_estimates(orc_ctx*, orc_match_t* best, double* p1p2 /*6 per estimate*/, long long cap);
long long orc_get_affinity(orc_ctx*, int* ei, int* ej, float* ew, long long cap); /* A_ handed to clustering */
long long orc_get_affinity_raw(orc_ctx*, int* ei, int* ej, float* ew, long long cap); /* A_ before diffusion */
int orc_get_local2global(orc_ctx*, uint32_t* cam_seg /*2 per id*/, int cap);
long long orc_get_collinear(orc_ctx*, uint32_t cam, long long* row_ptr, int* idx, long long cap); /* View::collin_ as CSR */
/* findCollinearSegments(cluster) (line3D.cc:2342-2452) on an explicit cluster of views added with orc_add_view */
int orc_collinear_from_cluster(orc_ctx*, const double* p1p2, int nres, const uint32_t* cams, const uint32_t* segs, double* out6, int cap);
int orc_num_lines(orc_ctx*);
long long orc_get_segments3d(orc_ctx*, orc_seg3d_t* out, long long cap);
long long orc_get_residuals(orc_ctx*, orc_residual_t* out, long long cap);
int orc_save_txt(orc_ctx*, const char* path);       /* save3DLinesAsTXT body (line3D.cc:2650-2681) */

#ifdef __cplusplus
}
#endif
#endif
