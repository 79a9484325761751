// l3d_ctx.cuh — the context object behind the opaque l3d_ctx* of include/l3d_capi.h
#pragma once
#include "l3d_match.cuh"

#include <algorithm>
#include <cstddef>
#include <memory>
#include <string>
#include <utility>
#include <vector>

// grow-only device allocation, freed with its owner
struct DevBuf {
    void* p = nullptr; size_t cap = 0;
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    DevBuf(DevBuf&& o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {}
    DevBuf& operator=(DevBuf&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); return *this; }
    ~DevBuf() { if (p) cudaFree(p); }
    int reserve(l3d_ctx* c, size_t bytes, const char* what);
};

// One caller array of a host-mode call: `rows` rows of `row_bytes` bytes, `pitch` bytes apart in host memory (a 1-D array is one
// row).  l3d_stage_host sets `dev` to the block's device copy: its rows packed (pitch row_bytes), starting on a 16-byte boundary.
struct HostBlock {
    const void* host;                       // an output block's array is written by l3d_unstage_host
    size_t pitch, row_bytes, rows;
    void* dev = nullptr;
};
inline HostBlock host_array(const void* p, size_t bytes) { return HostBlock{p, bytes, bytes, 1}; }

// Every caller's host array reaches the device here (host mode of the image, dense-matching and triangulation calls; the bundling,
// diffusion and argsort calls): packs the `in` blocks into the context's stage_in and the `out` blocks into its stage_out, uploads
// `in` on the context's stream and sets every block's dev.  l3d_unstage_host then downloads `out` from wherever its dev points and
// waits for the stream.  Two calls, so that a call may still fail in between and leave the caller's outputs untouched (the JPEG
// decode does when the coded data turns out corrupt).
int l3d_stage_host(l3d_ctx* c, HostBlock* in, int n_in, HostBlock* out, int n_out);
int l3d_unstage_host(l3d_ctx* c, const HostBlock* out, int n_out, const char* what);

// state of the per-view scoring sweep (l3d_pipeline.cu)
struct SweepState {
    bool valid = false;
    std::vector<int> order;                 // view indices in processing order (ascending camID)
    std::vector<long long> region_off;      // per processing rank (+1): first entry of the view's region
    long long total = 0;
    // match store (l3d_sweep.cuh): view table, chunk descriptors, chunk offsets, entries
    DevBuf d_vt, d_cinfo, d_rowoff, d_pinfo, d_bpair, d_ekv, d_rays, d_rmf, d_rflag, d_invpos, d_csize, d_ccur, d_cstart, d_eval, d_escore, d_eflag, d_gstage, d_gtab, d_export, d_export_ok,
        d_ranges, d_est_best, d_est_P, d_M, d_vmax, d_order, d_region_off, d_est_pos, d_est_out_best, d_est_out_P;
    long long n_est = 0;
    float ms_setup = 0.f, ms_chain = 0.f, ms_filter = 0.f;   // device time of the last sweep's three phases
};

// device state of the affinity matrix (l3d_affinity.cu), by step of l3d_affinity_matrix
struct AffinityState {
    bool valid = false; float two_sigA_sqr = 0.f, med = 0.f, min_aff = 0.f; long long K = 0, n_ids = 0;
    DevBuf d_kx;                                                                    // kept list
    DevBuf d_aff_sim, d_aff_flag, d_aff_gi, d_aff_gj, d_aff_cnt, d_evptr, d_aff_oi, d_aff_oj, d_aff_ow, d_aff_par;   // candidates
    DevBuf d_key, d_key2, d_val, d_val2, d_keep, d_keep2, d_found, d_changed;       // unused(): pair sort and fixpoint
    DevBuf d_q, d_time, d_nflag, d_npos, d_idof, d_nkey, d_nkey2, d_nval, d_nval2, d_l2g;   // appearance times and local ids
    DevBuf d_ei, d_ej, d_ew;                                                        // the emitted CLEdge list
};

// per-view lists of potentially collinear segments (l3d_collinear.cu), CSR over the global segment index
struct CollinState {
    bool valid = false; float dist_t = 0.f; int sem = 0; long long total = 0;
    DevBuf d_tiles, d_cnt, d_ptr, d_idx;
};

// device state of the line bundling (l3d_optimize.cu)
struct OptState {
    DevBuf d_obs, d_x, d_xc, d_g, d_H, d_S, d_diag, d_free, d_part, d_tot;
};

// device buffers of the diffusion (l3d_affinity.cu); d_idx and d_k2 are also the sort scratch of l3d_argsort_f32
struct RddState {
    DevBuf d_krow, d_kcol, d_k2, d_idx, d_idx2, d_P, d_Pn, d_W, d_prow, d_pcol, d_wmaj, d_wmin, d_rowptr, d_colptr, d_tslot, d_len4, d_rp4, d_cp4,
        d_Pp, d_Pnp, d_Wp, d_plan, d_dst;
};

// per-image parameters of the undistortion kernels (l3d_undistort.cu); ir0, ir2, ir4, ir5 = the non-trivial entries of
// inv([[fx',0,cx'],[0,fy',cy'],[0,0,1]]) of the new camera matrix (the camera's own K unless one is given); fx .. cy are the camera's
struct L3DUndistImage {
    const unsigned char* src;
    unsigned char* dst;
    const double* xcol;                      // fisheye: x of every output column (OpenCV's accumulated sum), in UndistortState::d_cols
    long long src_pitch, dst_pitch, tile0;   // tile0: first tile of this image in the batch grid
    int width, height, channels, tiles_x;    // width, height: the source (bounds the taps); tiles_x: of the output
    int kind;                                // lens kind of l3d_undistort.cu: radtan, radtan with k4..k6 (rational), fisheye
    int full_radial, tangential;             // 0: k2 = k3 = 0, resp. p1 = p2 = 0 (those terms are skipped)
    double ir0, ir2, ir4, ir5, fx, fy, cx, cy;
    double k1, k2, k3, k4, k5, k6, p1, p2;   // radtan: k1..k6, p1, p2; fisheye: k1..k4 are the theta coefficients
    int out_width, out_height;               // the output grid (the source size unless one is given)
};

// per-set parameters of k_undistort_points (l3d_undistort.cu): the camera, OpenCV's distortion vector and the new camera matrix
struct L3DPointSet {
    const float* src;
    float* dst;
    long long p0;                            // first point of this set in the batch
    double fx, fy, cx, cy, ifx, ify;         // the camera; ifx = 1 / fx, ify = 1 / fy (radtan multiplies by them, fisheye divides by f)
    double k[8];                             // radtan: OpenCV's k[0..7] = k1 k2 p1 p2 k3 k4 k5 k6; fisheye: k1..k4
    double nfx, nfy, ncx, ncy;               // the new camera matrix (the camera's own K unless one is given)
    int fisheye;
};

// buffers of the undistortion calls: not a pipeline stage, nothing else reads them
struct UndistortState {
    std::vector<L3DUndistImage> h_imgs;
    std::vector<double> h_cols;                          // fisheye column tables, one per distinct (ir0, ir2)
    std::vector<L3DPointSet> h_sets;                     // l3d_undistort_points
    DevBuf d_imgs, d_cols, d_sets;
};

// per-image parameters of k_prepare_gray_u8 (l3d_image_prep.cu): source (width x height, 1 or 3 channels) -> grey out_w x out_h
struct L3DPrepImage {
    const unsigned char* src;
    unsigned char* dst;
    long long src_pitch, dst_pitch, tile0;   // tile0: first tile of this image in the batch grid
    int width, height, channels, out_w, out_h, tiles_x;
    int mode;                                // L3D_PREP_COPY / L3D_PREP_LINEAR / L3D_PREP_AREA2
    double scale;                            // source step 1 / (double)s of the resize (OpenCV's scale_x = scale_y)
};

// buffers of the image preparation calls: not a pipeline stage, nothing else reads them
struct ImagePrepState {
    std::vector<L3DPrepImage> h_imgs;
    DevBuf d_imgs;
};

// a Huffman table as k_jpeg_entropy reads it (l3d_jpeg.cu): a 9-bit lookahead (length << 8 | symbol, 0 for a longer code), then
// libjpeg's canonical decode for lengths 10..16: a code c of length l is valid when c <= maxcode[l], its symbol vals[c + valoff[l]]
struct L3DJpegTable {
    unsigned short look[512];
    int maxcode[18], valoff[18];
    unsigned char vals[256];
};

// per-image parameters of the JPEG kernels (l3d_jpeg.cu)
struct L3DJpegImage {
    unsigned char* dst;
    long long dst_pitch, coef0, tile0;       // coef0: Y's first block in the coefficient buffer; tile0: first IDCT block in the batch grid
    int width, height, blocks_x;             // the coded frame; blocks_x: 8x8 blocks per row holding image pixels (ceil(width / 8))
    int yblocks_x;                           // Y's coded grid (MCU-padded in an interleaved scan)
    int ns, y_in_scan, mcus_x;               // Y's scan: components, Y's position, MCUs per row
    int bh[4], bv[4];                        // blocks of scan component k per MCU
    int ryy, ryx, ry0, rxy, rxx, rx0;        // EXIF orientation: the pixel (y, x) goes to row ryy*y + ryx*x + ry0, column rxy*y + rxx*x + rx0
    alignas(16) unsigned short q[64];        // Y's quantisation table, natural order (k_jpeg_idct reads it as uint4)
};
static_assert(offsetof(L3DJpegImage, q) % 16 == 0 && sizeof(L3DJpegImage) % 16 == 0, "L3DJpegImage::q is read as uint4");

// one entropy-coded segment: bytes [first, end) of the staged data, MCUs [mcu0, mcu1) of image `image`
struct L3DJpegSeg {
    long long first, end;
    int image, mcu0, mcu1, pad;
};

// buffers of the JPEG decode: not a pipeline stage, nothing else reads them
struct JpegState {
    std::vector<L3DJpegImage> h_imgs;
    std::vector<L3DJpegSeg> h_segs;
    std::vector<L3DJpegTable> h_tabs;                    // 8 per image: DC, AC of each component of Y's scan
    std::vector<int> h_status;
    DevBuf d_imgs, d_segs, d_tabs, d_bytes, d_coefs, d_status;
};

// per-image parameters of the PNG kernels (l3d_png.cu)
struct L3DPngImage {
    unsigned char* dst;
    long long dst_pitch, in0, in_len, raw0, raw_size, pix0;   // in0 / in_len: the zlib stream in d_in; raw0: the filtered rows in d_raw; pix0: first output pixel in the batch grid
    long long pass_off[7], pass_rb[7];       // per Adam7 pass: offset in the raw bytes, bytes per row (pass 0 only when not interlaced)
    int width, height, depth, color_type, channels, interlace, window;   // window: the zlib header's window in bytes
    int out_width, out_height, gamma;
    int ryy, ryx, ry0, rxy, rxx, rx0;        // EXIF orientation: the pixel (y, x) goes to row ryy*y + ryx*x + ry0, column rxy*y + rxx*x + rx0
    unsigned char palette[768], to_linear[256], from_linear[256];
};

// one Adam7 pass of one image for k_png_unfilter: rows of rb bytes (after the filter byte) at raw offset off, bpp bytes per unit
struct L3DPngPass {
    long long off;
    int image, rows, rb, bpp;
};

// buffers of the PNG decode: not a pipeline stage, nothing else reads them
struct PngState {
    std::vector<L3DPngImage> h_imgs;
    std::vector<L3DPngPass> h_passes;
    std::vector<unsigned char> h_in;                    // the batch's zlib streams, concatenated
    std::vector<int> h_status;
    DevBuf d_imgs, d_passes, d_in, d_raw, d_status;
};

// buffers of the median-depth call (l3d_triangulate.cu): not a pipeline stage either
struct TriangulateState {
    DevBuf d_keys, d_keys2;
};

// The results a context holds, each computed from the ones before it:
//   Views -> Matches -> Sweep -> Affinity,   Views -> Collinear -> Affinity
enum class Stage { Views, Matches, Sweep, Collinear, Affinity };

struct l3d_ctx {
    int device = 0, num_sms = 0;
    cudaStream_t stream = nullptr, copy_stream = nullptr;      // copy_stream: D2H of finished chunks (l3d_match_pairs_host)
    std::vector<cudaEvent_t> events;
    std::string err;
    long long launches = 0;
    DevBuf cub_tmp;                         // temporary storage of every cub call (all on `stream`, one at a time)
    DevBuf stage_in, stage_out;             // host-mode copies of the caller's arrays (l3d_stage_host), free again when the call returns

    // views
    bool have_views = false;
    int num_views = 0;
    long long total_segs = 0;
    std::vector<L3DViewDev> h_views;
    DevBuf d_segs, d_cache, d_cache_d, d_views;
    const float4* segs_ext = nullptr;       // caller-owned device segment array (l3d_set_views_flat on_device)
    std::unique_ptr<void, cudaError_t (*)(void*)> h_stage{nullptr, cudaFreeHost};    // pinned staging of l3d_set_views and of the device triples l3d_match_pairs_cand checks
    size_t h_stage_cap = 0;

    // last match result
    bool have_matches = false;
    int num_pairs = 0, knn = 0;             // knn: the row stride of d_recs
    int knn_asked = 0;                      // the kNN of the call (<= 0 as 0), which picks top-k or keep-all
    int first_pair = 0, last_pair = 0;      // the pairs evaluated: [first_pair, last_pair)
    float epi = 0.f;
    int semantics = 0;                      // L3D_SEM_* of the last match result; the scoring sweep follows it
    long long total_rows = 0, pair_evals = 0;
    std::vector<L3DPairDev> h_pairs;
    std::vector<int4> h_units;              // k_match_topk work units: (pair, first source row, rows, 0)
    DevBuf d_pairs, d_units, d_counts, d_recs, d_rowptr, d_csr, d_dense_jobs, d_arcs, d_basis, d_arcraw, d_arckeys, d_arckeys2, d_arcvals, d_arcvals2;
    DevBuf d_rowwin;                        // row windows of the rows of [level1_first, level1_last) (k_row_windows, L3D_RW_WORDS words per row)
    int level1_first = 0, level1_last = 0;  // the pairs whose level-1 tables, bases and row windows the context holds (its own last match call)
    // caller-given candidates of the last match call (l3d_match_pairs_cand): its per-pair restricted flags (empty: none), the restricted
    // pairs it evaluated as (pair, first restricted row), their rows in all (0: every pair scanned); on the device the per-pair flags,
    // those pairs, the triples (host mode), the sort's two key buffers (d_cand_keys: the sorted distinct keys) and their number
    std::vector<int> h_restricted;
    std::vector<longlong2> h_cand_pairs;
    long long cand_rows = 0;
    DevBuf d_restricted, d_cand_pairs, d_cand_trip, d_cand_keys, d_cand_keys2, d_cand_n;

    SweepState sweep;
    RddState rdd;
    AffinityState aff;
    CollinState collin;
    OptState opt;
    UndistortState undist;
    ImagePrepState prep;
    JpegState jpeg;
    PngState png;
    TriangulateState tri;

    const float4* segs() const { return segs_ext ? segs_ext : (const float4*)d_segs.p; }
    const L3DViewDev* views() const { return (const L3DViewDev*)d_views.p; }

    // Forget stage `s` and every stage computed from it.  An entry point that computes a stage drops it before it touches
    // any state and marks it present again only when it returns L3D_OK.
    void drop(Stage s)
    {
        switch (s) {
        case Stage::Views:     have_views = false; drop(Stage::Matches); drop(Stage::Collinear); break;
        case Stage::Matches:   have_matches = false; drop(Stage::Sweep); break;
        case Stage::Sweep:     sweep.valid = false; drop(Stage::Affinity); break;
        case Stage::Collinear: collin.valid = false; drop(Stage::Affinity); break;
        case Stage::Affinity:  aff.valid = false; break;
        }
    }
};

int l3d_fail(l3d_ctx* c, int code, const char* what, cudaError_t e = cudaSuccess);

#define L3D_CUDA(ctx, call, what)                                                     \
    do {                                                                              \
        cudaError_t _e = (call);                                                      \
        if (_e != cudaSuccess) return l3d_fail((ctx), L3D_ERR_CUDA, (what), _e);      \
    } while (0)

// grows `buf` to at least max(bytes, 16) bytes or returns the failure from the enclosing function (which declares `int rc`)
#define L3D_RESERVE(buf, bytes, what)                                                                             \
    do {                                                                                                          \
        if ((rc = (buf).reserve(c, (size_t)std::max<long long>((long long)(bytes), 16), (what)))) return rc;      \
    } while (0)

// CUDA event destroyed with its scope
struct ScopedEvent {
    cudaEvent_t e = nullptr;
    ScopedEvent() = default;
    ScopedEvent(const ScopedEvent&) = delete;
    ScopedEvent& operator=(const ScopedEvent&) = delete;
    ~ScopedEvent() { if (e) cudaEventDestroy(e); }
    int create(l3d_ctx* c) { L3D_CUDA(c, cudaEventCreate(&e), "event"); return L3D_OK; }
};
