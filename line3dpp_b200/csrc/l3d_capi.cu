// l3d_capi.cu — context, device memory and the C-ABI entry points declared in include/l3d_capi.h.
// Host C++ only orchestrates: every byte of arithmetic on the hot path runs in the kernels of l3d_match.cu /
// l3d_pipeline.cu.  There is no CPU fallback: every entry needs a live CUDA context and fails loudly otherwise.
#include "l3d_cub.cuh"
#include "l3d_sweep.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_reduce.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <cub/iterator/transform_input_iterator.cuh>

#include <algorithm>
#include <climits>
#include <cstdio>
#include <cstring>

int l3d_fail(l3d_ctx* c, int code, const char* what, cudaError_t e)
{
    if (c) {
        char buf[512];
        if (e != cudaSuccess) snprintf(buf, sizeof(buf), "%s: %s (%s)", what, cudaGetErrorName(e), cudaGetErrorString(e));
        else snprintf(buf, sizeof(buf), "%s", what);
        c->err = buf;
    }
    return code;
}

// The old allocation goes first, so that growing a large buffer never needs both sizes at once.  A failed reserve leaves the
// buffer empty; the stage it belongs to has been dropped by the entry point that reserves it.
int DevBuf::reserve(l3d_ctx* c, size_t bytes, const char* what)
{
    if (bytes <= cap) return L3D_OK;
    if (p) { cudaFree(p); p = nullptr; cap = 0; }
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) { e = cudaMalloc(&p, bytes); want = bytes; }
    if (e != cudaSuccess) { p = nullptr; return l3d_fail(c, L3D_ERR_NOMEM, what, e); }
    cap = want;
    return L3D_OK;
}

// the packed bytes of the blocks, each starting on a 16-byte boundary (k_remap_u8 reads its maps as short2 / ushort behind an image
// of any width, triangulation stages doubles, l3d_match_dense writes float4); with a base, also each block's dev
static size_t stage_layout(HostBlock* b, int n, char* base)
{
    size_t off = 0;
    for (int i = 0; i < n; ++i) {
        off = (off + 15) & ~(size_t)15;
        if (base) b[i].dev = base + off;
        off += b[i].row_bytes * b[i].rows;
    }
    return off;
}

int l3d_stage_host(l3d_ctx* c, HostBlock* in, int n_in, HostBlock* out, int n_out)
{
    int rc;
    L3D_RESERVE(c->stage_in, stage_layout(in, n_in, nullptr), "host-mode input staging");
    L3D_RESERVE(c->stage_out, stage_layout(out, n_out, nullptr), "host-mode output staging");
    stage_layout(in, n_in, (char*)c->stage_in.p);
    stage_layout(out, n_out, (char*)c->stage_out.p);
    for (int i = 0; i < n_in; ++i) {
        const HostBlock& b = in[i];
        if (b.row_bytes * b.rows == 0) continue;
        if (b.pitch == b.row_bytes) L3D_CUDA(c, cudaMemcpyAsync(b.dev, b.host, b.row_bytes * b.rows, cudaMemcpyHostToDevice, c->stream), "host-mode upload");
        else L3D_CUDA(c, cudaMemcpy2DAsync(b.dev, b.row_bytes, b.host, b.pitch, b.row_bytes, b.rows, cudaMemcpyHostToDevice, c->stream), "host-mode upload");
    }
    return L3D_OK;
}

int l3d_unstage_host(l3d_ctx* c, const HostBlock* out, int n_out, const char* what)
{
    for (int i = 0; i < n_out; ++i) {
        const HostBlock& b = out[i];
        void* host = const_cast<void*>(b.host);     // the caller's output array, writable
        if (b.row_bytes * b.rows == 0) continue;
        if (b.pitch == b.row_bytes) L3D_CUDA(c, cudaMemcpyAsync(host, b.dev, b.row_bytes * b.rows, cudaMemcpyDeviceToHost, c->stream), "host-mode download");
        else L3D_CUDA(c, cudaMemcpy2DAsync(host, b.pitch, b.dev, b.row_bytes, b.row_bytes, b.rows, cudaMemcpyDeviceToHost, c->stream), "host-mode download");
    }
    L3D_CUDA(c, cudaStreamSynchronize(c->stream), what);
    return L3D_OK;
}

struct CastI64 { __host__ __device__ long long operator()(int v) const { return (long long)v; } };

// the most dynamic shared memory k_sort_rows gets (run_keep_all: the rows of the CTA's warps at the keep-all stride)
static const size_t SORT_SMEM_MAX = 200 * 1024;
// the longest row a keep-all or kNN > 32 call can sort: one warp's row fills the block's shared memory (8533 matches)
static const int SORT_ROW_MAX = (int)(SORT_SMEM_MAX / sizeof(l3d_match_rec));

extern "C" {

int l3d_ctx_create(int device, l3d_ctx** out)
{
    if (!out) return L3D_ERR_INVALID;
    *out = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0 || device < 0 || device >= n) return L3D_ERR_CUDA;   // no GPU, no library: no CPU fallback
    l3d_ctx* c = new l3d_ctx();
    c->device = device;
    if ((e = cudaSetDevice(device)) != cudaSuccess || (e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking)) != cudaSuccess) {
        delete c;
        return L3D_ERR_CUDA;
    }
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, device);
    c->num_sms = prop.multiProcessorCount;
    for (int sem = 0; sem < 2; ++sem)
        for (auto k : l3d_match_kernels[sem])
            if (e == cudaSuccess) e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)l3d_match_smem_bytes(sem));
    // once, at the most any launch uses: the attribute is per device, and a per-launch setting would race between contexts that match
    // or score on one device from several host threads
    if (e == cudaSuccess) e = cudaFuncSetAttribute(k_sort_rows, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SORT_SMEM_MAX);
    for (int cpu_sem = 0; cpu_sem < 2; ++cpu_sem)
        for (auto k : l3d_sw_score_kernels[cpu_sem])
            if (e == cudaSuccess) e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)l3d_sw_score_smem_bytes(cpu_sem));
    if (e != cudaSuccess) { cudaStreamDestroy(c->stream); delete c; return L3D_ERR_CUDA; }
    *out = c;
    return L3D_OK;
}

void l3d_ctx_destroy(l3d_ctx* c)
{
    if (!c) return;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    for (cudaEvent_t e : c->events) cudaEventDestroy(e);
    if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
    cudaStreamDestroy(c->stream);
    delete c;
}

const char* l3d_last_error(const l3d_ctx* c) { return c ? c->err.c_str() : "null context"; }
void* l3d_stream(l3d_ctx* c) { return c ? (void*)c->stream : nullptr; }
long long l3d_launch_count(const l3d_ctx* c) { return c ? c->launches : 0; }
int l3d_sync(l3d_ctx* c)
{
    if (!c) return L3D_ERR_INVALID;
    cudaError_t e = cudaStreamSynchronize(c->stream);
    return e == cudaSuccess ? L3D_OK : l3d_fail(c, L3D_ERR_CUDA, "l3d_sync", e);
}

// ------------------------------------------------------------------------------------------------ views
static int set_views_common(l3d_ctx* c, int V, const l3d_view_desc* views)
{
    c->h_views.resize(V);
    long long off = 0;
    for (int v = 0; v < V; ++v) {
        if (views[v].nseg < 0) return l3d_fail(c, L3D_ERR_INVALID, "l3d_set_views: negative nseg");
        L3DViewDev& d = c->h_views[v];
        d.seg_off = off; d.nseg = views[v].nseg; d.cam_id = views[v].cam_id; d.width = views[v].width; d.height = views[v].height;
        memcpy(d.RtKinv, views[v].RtKinv, sizeof(d.RtKinv)); memcpy(d.C, views[v].C, sizeof(d.C));
        memcpy(d.RtKinv_d, views[v].RtKinv_d, sizeof(d.RtKinv_d)); memcpy(d.C_d, views[v].C_d, sizeof(d.C_d));
        d.k = views[v].k; d.median_depth = views[v].median_depth;
        off += views[v].nseg;
    }
    c->num_views = V; c->total_segs = off;
    return L3D_OK;
}

static int finish_views(l3d_ctx* c)
{
    int rc;
    if ((rc = c->d_views.reserve(c, sizeof(L3DViewDev) * (size_t)c->num_views, "views"))) return rc;
    if ((rc = c->d_cache.reserve(c, sizeof(float4) * 3 * (size_t)c->total_segs, "segment cache"))) return rc;
    L3D_CUDA(c, cudaMemcpyAsync(c->d_views.p, c->h_views.data(), sizeof(L3DViewDev) * c->num_views, cudaMemcpyHostToDevice, c->stream), "upload views");
    if (c->total_segs > 0) {
        unsigned int blocks = (unsigned int)((c->total_segs + 255) / 256);
        k_prep_segments<<<blocks, 256, 0, c->stream>>>(c->segs(), c->views(), c->num_views, c->total_segs, (float4*)c->d_cache.p);
        ++c->launches;
        L3D_CUDA(c, cudaGetLastError(), "k_prep_segments");
    }
    c->have_views = true;
    return L3D_OK;
}

int l3d_set_views(l3d_ctx* c, int V, const l3d_view_desc* views, const float* const* segs_host)
{
    if (!c) return L3D_ERR_INVALID;
    c->drop(Stage::Views);
    if (V <= 0 || !views || !segs_host) return l3d_fail(c, L3D_ERR_INVALID, "l3d_set_views: bad arguments");
    cudaSetDevice(c->device);
    int rc = set_views_common(c, V, views);
    if (rc) return rc;
    size_t bytes = sizeof(float4) * (size_t)c->total_segs;
    if ((rc = c->d_segs.reserve(c, bytes, "segments"))) return rc;
    if (bytes > c->h_stage_cap) {           // pinned staging so the H2D is one full-speed async copy
        void* p = nullptr;
        c->h_stage.reset(); c->h_stage_cap = 0;
        L3D_CUDA(c, cudaMallocHost(&p, bytes), "pinned staging");
        c->h_stage.reset(p); c->h_stage_cap = bytes;
    }
    L3D_CUDA(c, cudaStreamSynchronize(c->stream), "sync before staging");
    for (int v = 0; v < V; ++v)
        if (views[v].nseg) memcpy((char*)c->h_stage.get() + sizeof(float4) * c->h_views[v].seg_off, segs_host[v], sizeof(float4) * (size_t)views[v].nseg);
    if (bytes) L3D_CUDA(c, cudaMemcpyAsync(c->d_segs.p, c->h_stage.get(), bytes, cudaMemcpyHostToDevice, c->stream), "upload segments");
    c->segs_ext = nullptr;
    return finish_views(c);
}

int l3d_set_views_flat(l3d_ctx* c, int V, const l3d_view_desc* views, const float* segs_flat, int on_device)
{
    if (!c) return L3D_ERR_INVALID;
    c->drop(Stage::Views);
    if (V <= 0 || !views || !segs_flat) return l3d_fail(c, L3D_ERR_INVALID, "l3d_set_views_flat: bad arguments");
    cudaSetDevice(c->device);
    int rc = set_views_common(c, V, views);
    if (rc) return rc;
    size_t bytes = sizeof(float4) * (size_t)c->total_segs;
    if (on_device) {
        if (((uintptr_t)segs_flat & 15) != 0) return l3d_fail(c, L3D_ERR_INVALID, "l3d_set_views_flat: device array must be 16-byte aligned");
        c->segs_ext = (const float4*)segs_flat;
    } else {
        if ((rc = c->d_segs.reserve(c, bytes, "segments"))) return rc;
        if (bytes) L3D_CUDA(c, cudaMemcpyAsync(c->d_segs.p, segs_flat, bytes, cudaMemcpyHostToDevice, c->stream), "upload segments");
        c->segs_ext = nullptr;
    }
    return finish_views(c);
}

// new camera blocks for the same views: the matches and the sweep stay usable, the affinity matrix is recomputed
int l3d_update_view_params(l3d_ctx* c, int V, const l3d_view_desc* views)
{
    if (!c) return L3D_ERR_INVALID;
    c->drop(Stage::Affinity);
    if (!views || V != c->num_views || !c->have_views) return l3d_fail(c, L3D_ERR_STATE, "l3d_update_view_params: views not set / count mismatch");
    cudaSetDevice(c->device);
    L3D_CUDA(c, cudaStreamSynchronize(c->stream), "sync before view update");
    for (int v = 0; v < V; ++v) {
        L3DViewDev& d = c->h_views[v];
        memcpy(d.RtKinv_d, views[v].RtKinv_d, sizeof(d.RtKinv_d)); memcpy(d.C_d, views[v].C_d, sizeof(d.C_d));
        d.k = views[v].k; d.median_depth = views[v].median_depth;
    }
    const cudaError_t e = cudaMemcpyAsync(c->d_views.p, c->h_views.data(), sizeof(L3DViewDev) * V, cudaMemcpyHostToDevice, c->stream);
    if (e != cudaSuccess) { c->drop(Stage::Views); return l3d_fail(c, L3D_ERR_CUDA, "upload views", e); }   // host and device views differ
    return L3D_OK;
}

// ------------------------------------------------------------------------------------------------ matching
int l3d_match_pairs(l3d_ctx* c, int num_pairs, const int32_t* pairs, const float* F, float epi_overlap, int knn)
{ return l3d_match_pairs_range(c, num_pairs, pairs, F, epi_overlap, knn, 0, num_pairs); }

struct HostOut { int32_t* counts; l3d_match_rec* recs; int chunks; };
// Checks the arguments, fills h_pairs and the work units of k_match_topk for the pairs [first_pair, last_pair), uploads both and sizes the result buffers.
// *narcs: the number of level-1 table entries of the matched pairs.
// restricted (null: none): the per-pair flags of l3d_match_pairs_cand; a restricted pair has no level-1 table and no work units, its
// rows go to k_match_cand (h_cand_pairs) and its evaluations are counted by stage_candidates.
static int stage_pairs(l3d_ctx* c, int num_pairs, const int32_t* pairs, const float* F, const double* Fd, float epi_overlap, int knn,
                       int first_pair, int last_pair, const HostOut* host, const int32_t* restricted, long long* narcs)
{
    if (host && (!host->counts || !host->recs || host->chunks < 1)) return l3d_fail(c, L3D_ERR_INVALID, "l3d_match_pairs_host: bad arguments");
    if (host && knn <= 0) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_match_pairs_host: kNN <= 0 has no fixed row stride; use l3d_match_pairs + l3d_get_pair_matches");
    if (!c->have_views) return l3d_fail(c, L3D_ERR_STATE, "l3d_match_pairs: call l3d_set_views first");
    if (num_pairs < 0 || (num_pairs && (!pairs || (!F && !Fd)))) return l3d_fail(c, L3D_ERR_INVALID, "l3d_match_pairs: bad arguments");
    if (first_pair < 0 || last_pair < first_pair || last_pair > num_pairs) return l3d_fail(c, L3D_ERR_INVALID, "l3d_match_pairs_range: bad pair range");
    if (knn > 32 && host) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_match_pairs_host: kNN > 32 has no fixed row stride; use l3d_match_pairs + l3d_get_pair_matches");
    cudaSetDevice(c->device);
    L3D_CUDA(c, cudaStreamSynchronize(c->stream), "sync before pair staging");   // h_pairs/h_units may still be in flight
    c->h_pairs.resize(num_pairs);
    c->h_units.clear();
    c->h_cand_pairs.clear(); c->cand_rows = 0;
    if (restricted) c->h_restricted.assign(restricted, restricted + num_pairs); else c->h_restricted.clear();
    long long rows = 0, evals = 0;
    for (int i = 0; i < num_pairs; ++i) {
        int s = pairs[2 * i], t = pairs[2 * i + 1];
        if (s < 0 || t < 0 || s >= c->num_views || t >= c->num_views) return l3d_fail(c, L3D_ERR_INVALID, "l3d_match_pairs: view index out of range");
        L3DPairDev& p = c->h_pairs[i];
        p.src = s; p.tgt = t; p.row_off = rows;
        if (Fd) {     // REF_CPU: the double matrix decides; the float copy (eigen2dataArray-style cast) only feeds the conservative filter
            memcpy(p.Fd, Fd + 9 * (size_t)i, sizeof(p.Fd));
            for (int k = 0; k < 9; ++k) p.F[k] = (float)p.Fd[k];
        } else { memcpy(p.F, F + 9 * (size_t)i, sizeof(p.F)); memset(p.Fd, 0, sizeof(p.Fd)); }
        int Ns = c->h_views[s].nseg, Nt = c->h_views[t].nseg;
        if (Nt >= (1 << 24)) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_match_pairs: more than 2^24 segments in one view");
        p.arc_off = *narcs;
        const bool here = i >= first_pair && i < last_pair, scan = here && !(restricted && restricted[i]);
        if (here && !scan && Ns > 0) { c->h_cand_pairs.push_back(make_longlong2(i, c->cand_rows)); c->cand_rows += Ns; }
        if (scan) *narcs += Nt;
        if (Nt > 0 && scan) {     // the pair's rows in even units; several passes keep every row's list in a slot
            const int most = Nt <= MK_STAGES * MK_TT ? MK_UNIT_ROWS : MK_NSLOT, n = (Ns + most - 1) / most;
            for (int u = 0; u < n; ++u) {
                const int r0 = (int)((long long)Ns * u / n), r1 = (int)((long long)Ns * (u + 1) / n);
                c->h_units.push_back(make_int4(i, r0, r1 - r0, 0));
            }
        }
        rows += Ns;
        if (scan) evals += (long long)Ns * Nt;     // evaluated HERE
    }
    c->num_pairs = num_pairs; c->knn = knn; c->epi = epi_overlap; c->total_rows = rows; c->pair_evals = evals;
    c->knn_asked = std::max(knn, 0); c->first_pair = first_pair; c->last_pair = last_pair;
    int rc;
    L3D_RESERVE(c->d_pairs, sizeof(L3DPairDev) * (size_t)std::max(num_pairs, 1), "pairs");
    L3D_RESERVE(c->d_units, sizeof(int4) * std::max<size_t>(c->h_units.size(), 1), "tiles");
    L3D_RESERVE(c->d_arcs, (sizeof(uint4) + sizeof(float4)) * (size_t)std::max<long long>(*narcs, 1), "target arcs");   // arcs, then their segments
    L3D_RESERVE(c->d_basis, sizeof(L3DPairBasis) * (size_t)std::max(num_pairs, 1), "pair bases");
    L3D_RESERVE(c->d_counts, sizeof(int) * (size_t)std::max<long long>(rows, 1), "match counts");
    if (knn > 0 && knn <= 32) L3D_RESERVE(c->d_recs, sizeof(l3d_match_rec) * (size_t)std::max<long long>(rows, 1) * knn, "match records");
    if (num_pairs) L3D_CUDA(c, cudaMemcpyAsync(c->d_pairs.p, c->h_pairs.data(), sizeof(L3DPairDev) * num_pairs, cudaMemcpyHostToDevice, c->stream), "upload pairs");
    if (!c->h_units.empty()) L3D_CUDA(c, cudaMemcpyAsync(c->d_units.p, c->h_units.data(), sizeof(int4) * c->h_units.size(), cudaMemcpyHostToDevice, c->stream), "upload tiles");
    if (rows) L3D_CUDA(c, cudaMemsetAsync(c->d_counts.p, 0, sizeof(int) * rows, c->stream), "clear counts");   // rows of pairs with Nt == 0
    return L3D_OK;
}

// d_arcs holds the narcs packed arcs, then the target segment of every arc in the same order
static float4* level1_segs(l3d_ctx* c, long long narcs) { return (float4*)((uint4*)c->d_arcs.p + narcs); }

// Level-1 tables of the pairs matched here (l3d_device.cuh "pencil parameter"): raw arcs + keys, one sort, packed arcs and their target
// segments in window order.  Below epi_overlap 0.01 the extended arcs would span the whole line: everything is then handed to the float filter.
// restricted (device, null: none): pairs restricted to caller-given candidates get empty tables.
static int build_level1(l3d_ctx* c, int first_pair, int last_pair, long long narcs, float epi_overlap, const int* restricted)
{
    c->level1_first = c->level1_last = 0;
    if (last_pair <= first_pair || narcs <= 0) return L3D_OK;
    if (narcs >= (1ll << 31) - 2) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_match_pairs: more than 2^31 (pair, target segment) combinations in one call");
    const int npr = last_pair - first_pair;
    const bool on = epi_overlap >= 0.01f && getenv("L3D_NO_LEVEL1") == nullptr;
    int end_bit = 36;                       // key = pair << 36 | class << 32 | start of the arc
    while (end_bit < 64 && (1ll << (end_bit - 36)) < npr) ++end_bit;
    int rc;
    L3D_RESERVE(c->d_arcraw, 16 * narcs, "raw arcs"); L3D_RESERVE(c->d_arckeys, 8 * narcs, "arc keys"); L3D_RESERVE(c->d_arckeys2, 8 * narcs, "arc keys");
    L3D_RESERVE(c->d_arcvals, 4 * narcs, "arc order"); L3D_RESERVE(c->d_arcvals2, 4 * narcs, "arc order");
    k_pair_arcs<<<(unsigned int)npr, 256, 0, c->stream>>>(c->segs(), c->views(), (const L3DPairDev*)c->d_pairs.p, first_pair, on ? 1 : 0,
                                                         1.0 / (double)std::max(epi_overlap, 0.01f) + 0.5, restricted, (uint4*)c->d_arcraw.p,
                                                         (unsigned long long*)c->d_arckeys.p, (unsigned int*)c->d_arcvals.p, (L3DPairBasis*)c->d_basis.p);
    L3D_CUDA(c, cudaGetLastError(), "k_pair_arcs");
    if ((rc = l3d_cub(c, "arc sort", [&](void* tmp, size_t& bytes) {
             return cub::DeviceRadixSort::SortPairs(tmp, bytes, (const unsigned long long*)c->d_arckeys.p, (unsigned long long*)c->d_arckeys2.p,
                                                    (const unsigned int*)c->d_arcvals.p, (unsigned int*)c->d_arcvals2.p, (int)narcs, 0, end_bit, c->stream); }))) return rc;
    k_arcs_gather<<<(unsigned int)((narcs + 255) / 256), 256, 0, c->stream>>>(narcs, (const unsigned long long*)c->d_arckeys2.p, (const unsigned int*)c->d_arcvals2.p,
                                                                             (const uint4*)c->d_arcraw.p, c->segs(), c->views(), (const L3DPairDev*)c->d_pairs.p,
                                                                             first_pair, (uint4*)c->d_arcs.p, level1_segs(c, narcs));
    L3D_CUDA(c, cudaGetLastError(), "k_arcs_gather");
    c->launches += 2 + 8;
    // the row windows of every work unit, read by each k_match_topk launch of the call (all chunks of l3d_match_pairs_host)
    const long long row0 = c->h_pairs[first_pair].row_off, row1 = last_pair < c->num_pairs ? c->h_pairs[last_pair].row_off : c->total_rows;
    int stage = 0;
    for (int i = first_pair; i < last_pair; ++i) stage = std::max(stage, std::min(c->h_views[c->h_pairs[i].tgt].nseg, L3D_RW_STAGE));
    L3D_RESERVE(c->d_rowwin, 4 * L3D_RW_WORDS * (size_t)std::max<long long>(row1 - row0, 1), "row windows");
    if (!c->h_units.empty()) {
        k_row_windows<<<(unsigned int)c->h_units.size(), 256, sizeof(unsigned int) * (size_t)stage, c->stream>>>(
            c->segs(), c->views(), (const L3DPairDev*)c->d_pairs.p, (const int4*)c->d_units.p, (const L3DPairBasis*)c->d_basis.p,
            (const uint4*)c->d_arcs.p, row0, (uint4*)c->d_rowwin.p);
        ++c->launches;
        L3D_CUDA(c, cudaGetLastError(), "k_row_windows");
    }
    c->level1_first = first_pair; c->level1_last = last_pair;
    return L3D_OK;
}

// matchingCPU's rays / plane normals in double (REF_CPU); the camera blocks may have been updated since set_views
static int build_cache_d(l3d_ctx* c)
{
    if (c->total_segs == 0) return L3D_OK;
    int rc;
    L3D_RESERVE(c->d_cache_d, sizeof(double) * 9 * (size_t)c->total_segs, "double segment cache");
    k_prep_segments_f64<<<(unsigned int)((c->total_segs + 255) / 256), 256, 0, c->stream>>>(c->segs(), c->views(), c->num_views, c->total_segs, (double*)c->d_cache_d.p);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_prep_segments_f64");
    return L3D_OK;
}

// one launch of k_match_topk<c->semantics, keep> over the work units [t0, t1)
static int launch_match(l3d_ctx* c, Keep keep, MatchArgs a, size_t t0, size_t t1, const char* what)
{
    a.units += t0;
    void* args[] = {&a};
    cudaLaunchKernel((const void*)l3d_match_kernels[c->semantics][(int)keep], dim3((unsigned int)(t1 - t0)), dim3(MK_THREADS), args, l3d_match_smem_bytes(c->semantics), c->stream);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), what);
    return L3D_OK;
}

// one launch of k_match_cand<c->semantics, keep> over the restricted rows of the call (none: nothing)
static int launch_cand(l3d_ctx* c, Keep keep, CandArgs a, const char* what)
{
    if (c->cand_rows == 0) return L3D_OK;
    void* args[] = {&a};
    cudaLaunchKernel((const void*)l3d_cand_kernels[c->semantics][(int)keep], dim3((unsigned int)((c->cand_rows + CAND_WARPS - 1) / CAND_WARPS)),
                     dim3(32 * CAND_WARPS), args, 0, c->stream);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), what);
    return L3D_OK;
}

// The kNN best matches of every row: one launch, or (l3d_match_pairs_host) `chunks` launches over contiguous unit ranges with the D2H
// copy of every finished chunk's rows queued on a second stream, so that the PCIe transfer of chunk k hides behind the arithmetic of
// chunk k+1.
static int run_topk(l3d_ctx* c, const MatchArgs& a, const HostOut* host)
{
    const long long rows = c->total_rows, knn = a.knn;
    const size_t nunits = c->h_units.size();
    const int chunks = host ? std::max(1, std::min<int>(host->chunks, (int)std::max<size_t>(nunits, 1))) : 1;
    int rc;
    if (host) {
        if (!c->copy_stream) L3D_CUDA(c, cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking), "copy stream");
        while ((int)c->events.size() < chunks + 1) {
            cudaEvent_t e; L3D_CUDA(c, cudaEventCreateWithFlags(&e, cudaEventDisableTiming), "event");
            c->events.push_back(e);
        }
    }
    auto row_of_unit = [&](size_t t) { return t >= nunits ? rows : c->h_pairs[c->h_units[t].x].row_off + c->h_units[t].y; };
    long long row_done = 0;
    for (int k = 0; k < chunks; ++k) {
        const size_t t0 = nunits * (size_t)k / chunks, t1 = nunits * (size_t)(k + 1) / chunks;
        if (t1 > t0 && (rc = launch_match(c, Keep::TopK, a, t0, t1, "k_match_topk"))) return rc;
        if (host) {
            const long long r1 = k == chunks - 1 ? rows : row_of_unit(t1);      // rows [row_done, r1) are final after this launch
            if (r1 > row_done) {
                L3D_CUDA(c, cudaEventRecord(c->events[k], c->stream), "event record");
                L3D_CUDA(c, cudaStreamWaitEvent(c->copy_stream, c->events[k], 0), "event wait");
                L3D_CUDA(c, cudaMemcpyAsync(host->counts + row_done, (const int*)c->d_counts.p + row_done, sizeof(int) * (size_t)(r1 - row_done), cudaMemcpyDeviceToHost, c->copy_stream), "download counts");
                L3D_CUDA(c, cudaMemcpyAsync(host->recs + row_done * knn, (const l3d_match_rec*)c->d_recs.p + row_done * knn,
                                            sizeof(l3d_match_rec) * (size_t)(r1 - row_done) * knn, cudaMemcpyDeviceToHost, c->copy_stream), "download records");
                row_done = r1;
            }
        }
    }
    if (host) {     // the context's stream (the one callers time and synchronise) completes only after the last copy
        L3D_CUDA(c, cudaEventRecord(c->events[chunks], c->copy_stream), "event record");
        L3D_CUDA(c, cudaStreamWaitEvent(c->stream, c->events[chunks], 0), "event wait");
    }
    return L3D_OK;
}

// *out = the largest entry of the count array, at least 1 (the smallest stride a record array can have).  Waits for the stream.
static int row_max(l3d_ctx* c, int* out)
{
    const long long rows = c->total_rows;
    int rc, m = 0;
    if (rows > 0) {
        if (rows > INT_MAX) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_match_pairs: more than 2^31 rows with kNN <= 0");
        L3D_RESERVE(c->d_rowptr, 16, "row max");
        int* d_max = (int*)c->d_rowptr.p;
        if ((rc = l3d_cub(c, "row maximum", [&](void* tmp, size_t& bytes) {
                 return cub::DeviceReduce::Max(tmp, bytes, (const int*)c->d_counts.p, d_max, (int)rows, c->stream); }))) return rc;
        c->launches += 1;
        L3D_CUDA(c, cudaMemcpyAsync(&m, d_max, sizeof(int), cudaMemcpyDeviceToHost, c->stream), "row maximum");
        L3D_CUDA(c, cudaStreamSynchronize(c->stream), "sync");
    }
    *out = std::max(m, 1);
    return L3D_OK;
}

// The record array at `stride` slots per row in a new buffer: rows [a, z) are copied pitched (the first min(old, new) slots of each,
// no kernel), the others are left unset.  Waits for the copy, because the old buffer is freed on return.
static int relay_recs(l3d_ctx* c, int stride, long long a, long long z)
{
    const size_t REC = sizeof(l3d_match_rec);
    int rc;
    DevBuf out;
    if ((rc = out.reserve(c, REC * (size_t)std::max<long long>(c->total_rows, 1) * stride, "re-laid match records"))) return rc;
    if (z > a)
        L3D_CUDA(c, cudaMemcpy2DAsync((char*)out.p + REC * a * stride, REC * stride, (const char*)c->d_recs.p + REC * a * c->knn, REC * c->knn,
                                      REC * std::min(stride, c->knn), (size_t)(z - a), cudaMemcpyDeviceToDevice, c->stream), "re-lay match records");
    L3D_CUDA(c, cudaStreamSynchronize(c->stream), "re-lay match records");
    std::swap(c->d_recs, out);
    c->knn = stride;
    return L3D_OK;
}

// "Keep all matches" (kNN <= 0, cudawrapper.cu:628-636, line3D.cc:988-996): count pass -> row stride = largest row -> store pass ->
// rows sorted.  big_k > 0 (kNN > 32 exceeds the fused kernel's per-row key list): the same passes, and every row is cut to its big_k
// best afterwards (same matches as the reference's priority queue, line3D.cc:999-1006 / cudawrapper.cu:637-645).
// Restricted rows (l3d_match_pairs_cand) take the same passes in k_match_cand.
static int run_keep_all(l3d_ctx* c, MatchArgs a, int big_k, CandArgs ca)
{
    const long long rows = c->total_rows;
    const size_t nunits = c->h_units.size();
    const bool any = nunits || c->cand_rows;
    int rc, stride = 1;
    if (any) {
        a.knn = 0; a.recs = nullptr; ca.knn = 0; ca.recs = nullptr;
        if (nunits && (rc = launch_match(c, Keep::Count, a, 0, nunits, "k_match_topk (count)"))) return rc;
        if ((rc = launch_cand(c, Keep::Count, ca, "k_match_cand (count)"))) return rc;
        if ((rc = row_max(c, &stride))) return rc;
    }
    c->knn = stride;
    L3D_RESERVE(c->d_recs, sizeof(l3d_match_rec) * (size_t)std::max<long long>(rows, 1) * stride, "match records");
    if (any) {
        const size_t per_warp = sizeof(l3d_match_rec) * (size_t)stride;
        int wpb = 4;
        while (wpb > 1 && per_warp * wpb > SORT_SMEM_MAX) wpb >>= 1;
        if (stride > SORT_ROW_MAX) {
            char msg[120];
            snprintf(msg, sizeof(msg), "l3d_match_pairs: a row with more than %d matches (kNN <= 0 or kNN > 32)", SORT_ROW_MAX);
            return l3d_fail(c, L3D_ERR_UNSUPPORTED, msg);
        }
        a.knn = stride; a.recs = (l3d_match_rec*)c->d_recs.p; ca.knn = stride; ca.recs = a.recs;
        if (nunits && (rc = launch_match(c, Keep::Store, a, 0, nunits, "k_match_topk (store)"))) return rc;
        if ((rc = launch_cand(c, Keep::Store, ca, "k_match_cand (store)"))) return rc;
        const long long blocks = std::min<long long>((rows + wpb - 1) / wpb, (long long)c->num_sms * 16);
        k_sort_rows<<<(unsigned int)blocks, wpb * 32, per_warp * wpb, c->stream>>>((int*)c->d_counts.p, (l3d_match_rec*)c->d_recs.p, stride, rows, big_k);
        L3D_CUDA(c, cudaGetLastError(), "k_sort_rows");
        ++c->launches;
    }
    return L3D_OK;
}

// The triples of l3d_match_pairs_cand, checked on the host (a device array is read back first, into the context's pinned staging buffer):
// *ignored counts those of pairs that are not restricted or not evaluated here.  Needs the views; nothing is launched.
static int check_candidates(l3d_ctx* c, int num_pairs, const int32_t* pairs, const l3d_match_cand_desc* cand, const int32_t** trip,
                            int first_pair, int last_pair, long long* ignored)
{
    if (!cand || cand->n < 0 || (num_pairs > 0 && !cand->restricted) || (cand->n > 0 && !cand->triples))
        return l3d_fail(c, L3D_ERR_INVALID, "l3d_match_pairs_cand: null candidate descriptor or array, or n < 0");
    if (!c->have_views) return l3d_fail(c, L3D_ERR_STATE, "l3d_match_pairs: call l3d_set_views first");
    if (num_pairs < 0 || (num_pairs && !pairs)) return l3d_fail(c, L3D_ERR_INVALID, "l3d_match_pairs: bad arguments");
    if (cand->n >= INT_MAX) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_match_pairs_cand: 2^31 or more candidates in one call");
    *trip = cand->triples;
    if (cand->on_device && cand->n > 0) {
        cudaSetDevice(c->device);
        const size_t bytes = sizeof(int32_t) * 3 * (size_t)cand->n;
        if (bytes > c->h_stage_cap) {
            void* p = nullptr;
            L3D_CUDA(c, cudaStreamSynchronize(c->stream), "sync before staging");     // an upload of l3d_set_views may still read it
            c->h_stage.reset(); c->h_stage_cap = 0;
            L3D_CUDA(c, cudaMallocHost(&p, bytes), "pinned staging");
            c->h_stage.reset(p); c->h_stage_cap = bytes;
        }
        // on the context's stream: after whatever the caller queued there to fill the triples, before the kernels that read them
        L3D_CUDA(c, cudaMemcpyAsync(c->h_stage.get(), cand->triples, bytes, cudaMemcpyDeviceToHost, c->stream), "l3d_match_pairs_cand: read the candidates");
        L3D_CUDA(c, cudaStreamSynchronize(c->stream), "l3d_match_pairs_cand: read the candidates");
        *trip = (const int32_t*)c->h_stage.get();
    }
    std::vector<int2> seg_count((size_t)num_pairs);        // (Ns, Nt) of every pair
    for (int p = 0; p < num_pairs; ++p) {
        const int s = pairs[2 * p], t = pairs[2 * p + 1];
        if (s < 0 || t < 0 || s >= c->num_views || t >= c->num_views) return l3d_fail(c, L3D_ERR_INVALID, "l3d_match_pairs: view index out of range");
        seg_count[p] = make_int2(c->h_views[s].nseg, c->h_views[t].nseg);
    }
    *ignored = 0;
    for (long long k = 0; k < cand->n; ++k) {
        const int p = (*trip)[3 * k], a = (*trip)[3 * k + 1], b = (*trip)[3 * k + 2];
        char msg[200];
        if (p < 0 || p >= num_pairs) {
            snprintf(msg, sizeof(msg), "l3d_match_pairs_cand: candidate %lld names pair %d outside the pair list of %d", k, p, num_pairs);
            return l3d_fail(c, L3D_ERR_INVALID, msg);
        }
        const int Ns = seg_count[p].x, Nt = seg_count[p].y;
        if (a < 0 || a >= Ns || b < 0 || b >= Nt) {
            snprintf(msg, sizeof(msg), "l3d_match_pairs_cand: candidate %lld of pair %d: segment (%d, %d) outside the views' %d x %d segments", k, p, a, b, Ns, Nt);
            return l3d_fail(c, L3D_ERR_INVALID, msg);
        }
        *ignored += !(p >= first_pair && p < last_pair && cand->restricted[p]);
    }
    return L3D_OK;
}

// The candidates of the restricted pairs on the device: one key per triple (k_cand_keys), sorted, duplicates dropped (cub); k_match_cand
// finds a row's candidates by two binary searches.  *distinct: the distinct candidates of the restricted pairs evaluated here (waits).
static int stage_candidates(l3d_ctx* c, const l3d_match_cand_desc* cand, const int32_t* trip_host, int first_pair, int last_pair, long long ignored,
                            long long* distinct)
{
    const long long n = cand->n;
    int rc;
    if (c->total_rows >= (1ll << 39)) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_match_pairs_cand: 2^39 or more rows");
    L3D_RESERVE(c->d_cand_keys, 8 * n, "candidate keys"); L3D_RESERVE(c->d_cand_keys2, 8 * n, "candidate keys"); L3D_RESERVE(c->d_cand_n, sizeof(int), "candidate count");
    L3D_RESERVE(c->d_cand_pairs, sizeof(longlong2) * c->h_cand_pairs.size(), "restricted pairs");
    if (!c->h_cand_pairs.empty())
        L3D_CUDA(c, cudaMemcpyAsync(c->d_cand_pairs.p, c->h_cand_pairs.data(), sizeof(longlong2) * c->h_cand_pairs.size(), cudaMemcpyHostToDevice, c->stream), "upload restricted pairs");
    int nuniq = 0;
    if (n > 0) {
        const int32_t* trip = cand->triples;
        if (!cand->on_device) {
            L3D_RESERVE(c->d_cand_trip, sizeof(int32_t) * 3 * n, "candidates");
            L3D_CUDA(c, cudaMemcpyAsync(c->d_cand_trip.p, trip_host, sizeof(int32_t) * 3 * n, cudaMemcpyHostToDevice, c->stream), "upload candidates");
            trip = (const int32_t*)c->d_cand_trip.p;
        }
        k_cand_keys<<<(unsigned int)((n + 255) / 256), 256, 0, c->stream>>>(n, trip, (const L3DPairDev*)c->d_pairs.p, (const int*)c->d_restricted.p,
                                                                          first_pair, last_pair, (unsigned long long*)c->d_cand_keys2.p);
        L3D_CUDA(c, cudaGetLastError(), "k_cand_keys");
        if ((rc = l3d_cub(c, "candidate sort", [&](void* tmp, size_t& bytes) {
                 return cub::DeviceRadixSort::SortKeys(tmp, bytes, (const unsigned long long*)c->d_cand_keys2.p, (unsigned long long*)c->d_cand_keys.p,
                                                       (int)n, 0, 64, c->stream); }))) return rc;
        if ((rc = l3d_cub(c, "candidate dedup", [&](void* tmp, size_t& bytes) {
                 return cub::DeviceSelect::Unique(tmp, bytes, (const unsigned long long*)c->d_cand_keys.p, (unsigned long long*)c->d_cand_keys2.p,
                                                  (int*)c->d_cand_n.p, (int)n, c->stream); }))) return rc;
        std::swap(c->d_cand_keys, c->d_cand_keys2);
        c->launches += 1 + 4 + 1;
        L3D_CUDA(c, cudaMemcpyAsync(&nuniq, c->d_cand_n.p, sizeof(int), cudaMemcpyDeviceToHost, c->stream), "candidate count");
        L3D_CUDA(c, cudaStreamSynchronize(c->stream), "candidate count");
    } else L3D_CUDA(c, cudaMemsetAsync(c->d_cand_n.p, 0, sizeof(int), c->stream), "candidate count");
    *distinct = nuniq - (ignored > 0 ? 1 : 0);      // the ignored triples leave one L3D_CAND_NONE key, sorted last
    return L3D_OK;
}

static int match_impl(l3d_ctx* c, int num_pairs, const int32_t* pairs, const float* F, const double* Fd, float epi_overlap, int knn, int first_pair, int last_pair,
                      const HostOut* host = nullptr, const l3d_match_cand_desc* cand = nullptr, bool with_cand = false)
{
    if (!c) return L3D_ERR_INVALID;
    c->drop(Stage::Matches);
    int rc;
    long long narcs = 0, ignored = 0, distinct = 0;
    const int32_t* trip = nullptr;
    if (with_cand && (rc = check_candidates(c, num_pairs, pairs, cand, &trip, first_pair, last_pair, &ignored))) return rc;
    if ((rc = stage_pairs(c, num_pairs, pairs, F, Fd, epi_overlap, knn, first_pair, last_pair, host, with_cand ? cand->restricted : nullptr, &narcs))) return rc;
    if (with_cand) {
        L3D_RESERVE(c->d_restricted, sizeof(int) * (size_t)num_pairs, "restricted pairs");
        if (num_pairs) L3D_CUDA(c, cudaMemcpyAsync(c->d_restricted.p, cand->restricted, sizeof(int) * (size_t)num_pairs, cudaMemcpyHostToDevice, c->stream), "upload restricted pairs");
    }
    if ((rc = build_level1(c, first_pair, last_pair, narcs, epi_overlap, with_cand ? (const int*)c->d_restricted.p : nullptr))) return rc;
    if (with_cand && (rc = stage_candidates(c, cand, trip, first_pair, last_pair, ignored, &distinct))) return rc;
    c->pair_evals += distinct;
    if (Fd && (rc = build_cache_d(c))) return rc;
    c->semantics = Fd ? L3D_SEM_REF_CPU : L3D_SEM_REF_GPU;
    const MatchArgs a = {c->segs(), (const float4*)c->d_cache.p, Fd ? (const double*)c->d_cache_d.p : nullptr, c->views(), (const L3DPairDev*)c->d_pairs.p,
                         (const int4*)c->d_units.p, (const uint4*)c->d_arcs.p, level1_segs(c, narcs), (const L3DPairBasis*)c->d_basis.p,
                         (const uint4*)c->d_rowwin.p, first_pair < num_pairs ? c->h_pairs[first_pair].row_off : 0, (int*)c->d_counts.p,
                         (l3d_match_rec*)c->d_recs.p, knn, epi_overlap};
    const CandArgs ca = {a.segs, a.cache, a.cache_d, a.views, a.pairs, (const longlong2*)c->d_cand_pairs.p, (int)c->h_cand_pairs.size(), c->cand_rows,
                         (const unsigned long long*)c->d_cand_keys.p, (const int*)c->d_cand_n.p, a.counts, a.recs, knn, epi_overlap};
    if (knn > 0 && knn <= 32) {
        if ((rc = run_topk(c, a, host)) || (rc = launch_cand(c, Keep::TopK, ca, "k_match_cand"))) return rc;
    } else if ((rc = run_keep_all(c, a, knn > 32 ? knn : 0, ca))) return rc;
    c->have_matches = true;
    return L3D_OK;
}

int l3d_match_pairs_range(l3d_ctx* c, int num_pairs, const int32_t* pairs, const float* F, float epi_overlap, int knn, int first_pair, int last_pair)
{ return match_impl(c, num_pairs, pairs, F, nullptr, epi_overlap, knn, first_pair, last_pair); }

int l3d_match_pairs_f64(l3d_ctx* c, int num_pairs, const int32_t* pairs, const double* Fd, float epi_overlap, int knn, int first_pair, int last_pair)
{ return match_impl(c, num_pairs, pairs, nullptr, Fd, epi_overlap, knn, first_pair, last_pair); }

int l3d_match_pairs_cand(l3d_ctx* c, int num_pairs, const int32_t* pairs, const float* F, float epi_overlap, int knn, int first_pair, int last_pair,
                         const l3d_match_cand_desc* cand)
{ return match_impl(c, num_pairs, pairs, F, nullptr, epi_overlap, knn, first_pair, last_pair, nullptr, cand, true); }

int l3d_match_pairs_cand_f64(l3d_ctx* c, int num_pairs, const int32_t* pairs, const double* Fd, float epi_overlap, int knn, int first_pair,
                             int last_pair, const l3d_match_cand_desc* cand)
{ return match_impl(c, num_pairs, pairs, nullptr, Fd, epi_overlap, knn, first_pair, last_pair, nullptr, cand, true); }

int l3d_match_pairs_host(l3d_ctx* c, int num_pairs, const int32_t* pairs, const float* F, float epi_overlap, int knn, int32_t* counts_out,
                         l3d_match_rec* recs_out, int chunks)
{
    HostOut h = {counts_out, recs_out, std::min(chunks, 64)};
    return match_impl(c, num_pairs, pairs, F, nullptr, epi_overlap, knn, 0, num_pairs, &h);
}

int l3d_match_device_buffers(l3d_ctx* c, void** counts_dev, void** recs_dev)
{
    if (!c || !counts_dev || !recs_dev) return L3D_ERR_INVALID;
    if (!c->have_matches) return l3d_fail(c, L3D_ERR_STATE, "l3d_match_device_buffers: no match result");
    *counts_dev = c->d_counts.p; *recs_dev = c->d_recs.p;
    c->drop(Stage::Sweep);                  // the caller may overwrite rows
    return L3D_OK;
}

int l3d_match_row_windows(l3d_ctx* c, int pair, uint32_t* windows_out, double* basis_out, int32_t* class_off_out, uint32_t* arc_starts_out)
{
    if (!c) return L3D_ERR_INVALID;
    if (!c->have_matches) return l3d_fail(c, L3D_ERR_STATE, "l3d_match_row_windows: no match result");
    if (pair < c->level1_first || pair >= c->level1_last) return l3d_fail(c, L3D_ERR_INVALID, "l3d_match_row_windows: pair not evaluated by the last match call");
    if (!c->h_restricted.empty() && c->h_restricted[pair])
        return l3d_fail(c, L3D_ERR_INVALID, "l3d_match_row_windows: the pair was restricted to caller-given candidates: it has no level-1 table or row windows");
    cudaSetDevice(c->device);
    const L3DPairDev& p = c->h_pairs[pair];
    const int Ns = c->h_views[p.src].nseg, Nt = c->h_views[p.tgt].nseg;
    if (Nt == 0) return L3D_OK;             // no level-1 table and no windows: the pair has no candidates
    L3DPairBasis B;
    L3D_CUDA(c, cudaMemcpyAsync(&B, (const L3DPairBasis*)c->d_basis.p + pair, sizeof(B), cudaMemcpyDeviceToHost, c->stream), "download pair basis");
    if (windows_out && Ns)
        L3D_CUDA(c, cudaMemcpyAsync(windows_out, (const uint32_t*)c->d_rowwin.p + (p.row_off - c->h_pairs[c->level1_first].row_off) * L3D_RW_WORDS,
                                    4 * L3D_RW_WORDS * (size_t)Ns, cudaMemcpyDeviceToHost, c->stream), "download row windows");
    if (arc_starts_out)     // x of every packed entry (uint4) of the pair's sorted table
        L3D_CUDA(c, cudaMemcpy2DAsync(arc_starts_out, 4, (const uint4*)c->d_arcs.p + p.arc_off, sizeof(uint4), 4, (size_t)Nt, cudaMemcpyDeviceToHost, c->stream),
                 "download arc starts");
    L3D_CUDA(c, cudaStreamSynchronize(c->stream), "sync");
    if (basis_out) for (int i = 0; i < 3; ++i) { basis_out[i] = B.u[i]; basis_out[3 + i] = B.v[i]; }
    if (class_off_out) for (int i = 0; i < L3D_ARC_NCLS + 2; ++i) class_off_out[i] = B.cls_off[i];
    return L3D_OK;
}

int l3d_pair_row_offsets(l3d_ctx* c, long long* out)
{
    if (!c || !out) return L3D_ERR_INVALID;
    if (!c->have_matches) return l3d_fail(c, L3D_ERR_STATE, "l3d_pair_row_offsets: no match result");
    for (int i = 0; i < c->num_pairs; ++i) out[i] = c->h_pairs[i].row_off;
    out[c->num_pairs] = c->total_rows;
    return L3D_OK;
}

int l3d_balanced_split(const long long* cost, int n, int parts, int32_t* bounds)
{
    if (n < 0 || parts < 1 || !bounds || (n && !cost)) return L3D_ERR_INVALID;
    long long total = 0;
    for (int i = 0; i < n; ++i) { if (cost[i] < 0) return L3D_ERR_INVALID; total += cost[i]; }
    // item i goes to the part whose cost window contains the midpoint of i's cost interval: monotone, so ranges are contiguous
    bounds[0] = 0;
    int part = 0; long long before = 0;
    for (int i = 0; i < n; ++i) {
        const long double mid = (long double)before + 0.5L * (long double)cost[i];
        int want = total > 0 ? (int)(mid * parts / (long double)total) : (int)((long long)i * parts / n);
        if (want >= parts) want = parts - 1;
        while (part < want) bounds[++part] = i;
        before += cost[i];
    }
    while (part < parts) bounds[++part] = n;
    return L3D_OK;
}

}   // extern "C"

// ------------------------------------------------------------------------------------------------ gathering match rows
// whether s holds a match result of the same job as d: the same views' sizes, pairs, matrices, rows, semantics, epi and kNN request
static bool same_job(const l3d_ctx* d, const l3d_ctx* s)
{
    if (s->num_pairs != d->num_pairs || s->total_rows != d->total_rows || s->semantics != d->semantics || s->epi != d->epi ||
        s->knn_asked != d->knn_asked || s->num_views != d->num_views)
        return false;
    for (int v = 0; v < d->num_views; ++v)
        if (s->h_views[v].nseg != d->h_views[v].nseg) return false;
    for (int i = 0; i < d->num_pairs; ++i) {
        const L3DPairDev &a = d->h_pairs[i], &b = s->h_pairs[i];
        if (a.src != b.src || a.tgt != b.tgt || a.row_off != b.row_off || memcmp(a.F, b.F, sizeof(a.F)) || memcmp(a.Fd, b.Fd, sizeof(a.Fd))) return false;
    }
    return true;
}

static int gather_check(l3d_ctx* d, int n, l3d_ctx* const* src, const int32_t* b)
{
    char msg[160];
    if (n < 1 || !src || !b) return l3d_fail(d, L3D_ERR_INVALID, "l3d_match_gather: bad arguments");
    if (!d->have_matches) return l3d_fail(d, L3D_ERR_STATE, "l3d_match_gather: the destination has no match result");
    if (b[0] < 0 || b[n] > d->num_pairs) return l3d_fail(d, L3D_ERR_INVALID, "l3d_match_gather: pair bounds outside the pair list");
    for (int i = 0; i < n; ++i) {
        const l3d_ctx* s = src[i];
        if (!s || b[i + 1] < b[i]) return l3d_fail(d, L3D_ERR_INVALID, "l3d_match_gather: null source or decreasing pair bounds");
        if (!s->have_matches) {
            snprintf(msg, sizeof(msg), "l3d_match_gather: source %d has no match result", i);
            return l3d_fail(d, L3D_ERR_STATE, msg);
        }
        if (!same_job(d, s)) {
            snprintf(msg, sizeof(msg), "l3d_match_gather: source %d matched another pair list, semantics, epi or kNN", i);
            return l3d_fail(d, L3D_ERR_INVALID, msg);
        }
        if (s->first_pair != b[i] || s->last_pair != b[i + 1]) {
            snprintf(msg, sizeof(msg), "l3d_match_gather: source %d evaluated pairs [%d, %d), not [%d, %d)", i, s->first_pair, s->last_pair, b[i], b[i + 1]);
            return l3d_fail(d, L3D_ERR_INVALID, msg);
        }
    }
    return L3D_OK;
}

// the first row of pair p, total_rows for p == num_pairs
static long long row_of_pair(const l3d_ctx* c, int p) { return p < c->num_pairs ? c->h_pairs[p].row_off : c->total_rows; }

static cudaError_t copy_rows(l3d_ctx* d, void* dp, const l3d_ctx* s, const void* sp, size_t bytes)
{
    return s->device == d->device ? cudaMemcpyAsync(dp, sp, bytes, cudaMemcpyDeviceToDevice, d->stream)
                                  : cudaMemcpyPeerAsync(dp, d->device, sp, s->device, bytes, d->stream);
}

// `height` rows of `width` bytes from a pitch of spitch to one of dpitch
static cudaError_t copy_pitched(l3d_ctx* d, void* dp, size_t dpitch, const l3d_ctx* s, const void* sp, size_t spitch, size_t width, size_t height)
{
    if (s->device == d->device) return cudaMemcpy2DAsync(dp, dpitch, sp, spitch, width, height, cudaMemcpyDeviceToDevice, d->stream);
    cudaMemcpy3DPeerParms p = {};
    p.srcPtr = make_cudaPitchedPtr(const_cast<void*>(sp), spitch, width, height); p.srcDevice = s->device;
    p.dstPtr = make_cudaPitchedPtr(dp, dpitch, width, height); p.dstDevice = d->device;
    p.extent = make_cudaExtent(width, height, 1);
    return cudaMemcpy3DPeerAsync(&p, d->stream);
}

// direct copies from `peer` where the hardware allows it; otherwise cudaMemcpyPeerAsync stages through the host.  Peer access is state of
// this process's runtime, not a device setting.  The current device is d's.
static int enable_peer(l3d_ctx* d, int peer)
{
    int can = 0;
    L3D_CUDA(d, cudaDeviceCanAccessPeer(&can, d->device, peer), "cudaDeviceCanAccessPeer");
    if (!can) return L3D_OK;
    const cudaError_t e = cudaDeviceEnablePeerAccess(peer, 0);
    if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); return L3D_OK; }
    L3D_CUDA(d, e, "cudaDeviceEnablePeerAccess");
    return L3D_OK;
}

// d's stream waits until s's stream has passed everything enqueued so far (s's match result is complete)
static int wait_for(l3d_ctx* d, l3d_ctx* s)
{
    cudaEvent_t ev;
    cudaSetDevice(s->device);
    cudaError_t e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    if (e == cudaSuccess) {
        e = cudaEventRecord(ev, s->stream);
        cudaSetDevice(d->device);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(d->stream, ev, 0);
        cudaEventDestroy(ev);               // released once the wait has passed it
    }
    cudaSetDevice(d->device);
    L3D_CUDA(d, e, "l3d_match_gather: wait for a source");
    return L3D_OK;
}

// The rows [row_of_pair(b[0]), row_of_pair(b[n])) from their sources, at the stride one context matching all those pairs would have
// chosen: kNN for top-k; for keep-all the longest row, i.e. the largest of the sources' strides.  Rows outside get count 0.
static int gather_rows(l3d_ctx* d, int n, l3d_ctx* const* src, const int32_t* b)
{
    cudaSetDevice(d->device);
    const size_t REC = sizeof(l3d_match_rec);
    const bool topk = d->knn_asked >= 1 && d->knn_asked <= 32;
    int stride = topk ? d->knn_asked : 1, rc;
    bool d_is_src = false;
    for (int i = 0; i < n; ++i) { stride = std::max(stride, src[i]->knn); d_is_src |= src[i] == d; }
    if (!topk && stride != d->knn) {
        if (d_is_src) {     // re-lay d's own rows at the wider stride (d's stride is one of the maximum's terms, so it is the smaller)
            if ((rc = relay_recs(d, stride, row_of_pair(d, d->first_pair), row_of_pair(d, d->last_pair)))) return rc;
        } else {
            if ((rc = d->d_recs.reserve(d, REC * (size_t)std::max<long long>(d->total_rows, 1) * stride, "gathered match records"))) return rc;
            d->knn = stride;
        }
    }
    const long long r0 = row_of_pair(d, b[0]), r1 = row_of_pair(d, b[n]);
    if (r0 > 0) L3D_CUDA(d, cudaMemsetAsync(d->d_counts.p, 0, sizeof(int) * r0, d->stream), "clear counts");
    if (r1 < d->total_rows) L3D_CUDA(d, cudaMemsetAsync((int*)d->d_counts.p + r1, 0, sizeof(int) * (d->total_rows - r1), d->stream), "clear counts");
    for (int i = 0; i < n; ++i) {
        l3d_ctx* s = src[i];
        const long long a = row_of_pair(d, b[i]), z = row_of_pair(d, b[i + 1]);
        if (s == d || z <= a) continue;
        if (s->device != d->device && (rc = enable_peer(d, s->device))) return rc;
        if ((rc = wait_for(d, s))) return rc;
        L3D_CUDA(d, copy_rows(d, (int*)d->d_counts.p + a, s, (const int*)s->d_counts.p + a, sizeof(int) * (size_t)(z - a)), "l3d_match_gather: copy counts");
        char* dr = (char*)d->d_recs.p + REC * a * stride;
        const char* sr = (const char*)s->d_recs.p + REC * a * s->knn;
        L3D_CUDA(d, s->knn == stride ? copy_rows(d, dr, s, sr, REC * stride * (size_t)(z - a))
                                     : copy_pitched(d, dr, REC * stride, s, sr, REC * s->knn, REC * s->knn, (size_t)(z - a)),
                 "l3d_match_gather: copy records");
    }
    long long evals = 0;                    // each source's own count: Ns*Nt per scanned pair, the distinct candidates of a restricted one
    for (int i = 0; i < n; ++i) evals += src[i]->pair_evals;
    d->pair_evals = evals; d->first_pair = b[0]; d->last_pair = b[n];
    return L3D_OK;
}

extern "C" {

int l3d_match_gather(l3d_ctx* dst, int n_src, l3d_ctx* const* src, const int32_t* pair_bounds)
{
    if (!dst) return L3D_ERR_INVALID;
    int rc = gather_check(dst, n_src, src, pair_bounds);
    dst->drop(Stage::Matches);              // also on success: the rows change under the sweep and what follows it
    if (rc || (rc = gather_rows(dst, n_src, src, pair_bounds))) return rc;
    dst->have_matches = true;
    return L3D_OK;
}

static int restride(l3d_ctx* c, int stride)
{
    cudaSetDevice(c->device);
    const long long SLOTS = 1ll << 31;      // the scoring sweep indexes record slots in 32 bits (l3d_score_sweep)
    const char* too_many = "l3d_match_restride: 2^31 or more record slots";
    if (c->total_rows >= SLOTS) return l3d_fail(c, L3D_ERR_INVALID, too_many);
    int longest, rc;
    if ((rc = row_max(c, &longest))) return rc;
    if (stride <= 0) stride = longest;
    if (stride < longest) {
        char msg[128];
        snprintf(msg, sizeof(msg), "l3d_match_restride: stride %d is below the longest row (%d matches)", stride, longest);
        return l3d_fail(c, L3D_ERR_INVALID, msg);
    }
    if (c->total_rows * stride >= SLOTS) return l3d_fail(c, L3D_ERR_INVALID, too_many);
    return stride == c->knn ? L3D_OK : relay_recs(c, stride, 0, c->total_rows);
}

int l3d_match_restride(l3d_ctx* c, int stride)
{
    if (!c) return L3D_ERR_INVALID;
    if (!c->have_matches) return l3d_fail(c, L3D_ERR_STATE, "l3d_match_restride: no match result");
    c->drop(Stage::Matches);                // the rows move under the sweep and what follows it
    const int rc = restride(c, stride);
    if (rc) return rc;
    c->have_matches = true;
    return c->knn;
}

int l3d_match_stride(const l3d_ctx* c) { return c && c->have_matches ? c->knn : L3D_ERR_STATE; }
int l3d_match_semantics(const l3d_ctx* c) { return c && c->have_matches ? c->semantics : L3D_ERR_STATE; }
long long l3d_match_total_rows(const l3d_ctx* c) { return c && c->have_matches ? c->total_rows : -1; }
long long l3d_match_pair_evals(const l3d_ctx* c) { return c && c->have_matches ? c->pair_evals : -1; }

long long l3d_get_match_counts(l3d_ctx* c, int32_t* counts_out)
{
    if (!c || !counts_out) return L3D_ERR_INVALID;
    if (!c->have_matches) return l3d_fail(c, L3D_ERR_STATE, "l3d_get_match_counts: no match result");
    cudaSetDevice(c->device);
    if (c->total_rows) {
        cudaError_t e = cudaMemcpyAsync(counts_out, c->d_counts.p, sizeof(int) * c->total_rows, cudaMemcpyDeviceToHost, c->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
        if (e != cudaSuccess) return l3d_fail(c, L3D_ERR_CUDA, "download counts", e);
    }
    long long total = 0;
    for (long long i = 0; i < c->total_rows; ++i) total += counts_out[i];
    return total;
}

// number of matches of the last match result (sum of the per-row counts), reduced on the device: no download of the count array
long long l3d_match_total_matches(l3d_ctx* c)
{
    if (!c) return L3D_ERR_INVALID;
    if (!c->have_matches) return l3d_fail(c, L3D_ERR_STATE, "l3d_match_total_matches: no match result");
    if (c->total_rows == 0) return 0;
    cudaSetDevice(c->device);
    int rc;
    long long total = 0;
    const long long BLK = 1ll << 30;
    L3D_RESERVE(c->d_rowptr, 16, "match total");
    for (long long base = 0; base < c->total_rows; base += BLK) {
        const int n = (int)std::min(BLK, c->total_rows - base);
        long long part = 0;
        if ((rc = l3d_cub(c, "match total", [&](void* tmp, size_t& bytes) {
                 return cub::DeviceReduce::Sum(tmp, bytes, (const int*)c->d_counts.p + base, (long long*)c->d_rowptr.p, n, c->stream); }))) return rc;
        L3D_CUDA(c, cudaMemcpyAsync(&part, c->d_rowptr.p, 8, cudaMemcpyDeviceToHost, c->stream), "match total");
        L3D_CUDA(c, cudaStreamSynchronize(c->stream), "match total");
        total += part;
        ++c->launches;
    }
    return total;
}

int l3d_get_pair_matches(l3d_ctx* c, int pair, int32_t* counts_out, l3d_match_rec* recs_out)
{
    if (!c || !counts_out || !recs_out) return L3D_ERR_INVALID;
    if (!c->have_matches) return l3d_fail(c, L3D_ERR_STATE, "l3d_get_pair_matches: no match result");
    if (pair < 0 || pair >= c->num_pairs) return l3d_fail(c, L3D_ERR_INVALID, "l3d_get_pair_matches: pair out of range");
    cudaSetDevice(c->device);
    const L3DPairDev& p = c->h_pairs[pair];
    int Ns = c->h_views[p.src].nseg;
    if (Ns == 0) return L3D_OK;
    L3D_CUDA(c, cudaMemcpyAsync(counts_out, (const int*)c->d_counts.p + p.row_off, sizeof(int) * Ns, cudaMemcpyDeviceToHost, c->stream), "download pair counts");
    L3D_CUDA(c, cudaMemcpyAsync(recs_out, (const l3d_match_rec*)c->d_recs.p + p.row_off * c->knn, sizeof(l3d_match_rec) * (size_t)Ns * c->knn, cudaMemcpyDeviceToHost, c->stream), "download pair records");
    L3D_CUDA(c, cudaStreamSynchronize(c->stream), "sync");
    return L3D_OK;
}

long long l3d_get_matches_csr(l3d_ctx* c, int64_t* row_ptr_out, l3d_match_rec* recs_out, long long capacity)
{
    if (!c || !row_ptr_out) return L3D_ERR_INVALID;
    if (!c->have_matches) return l3d_fail(c, L3D_ERR_STATE, "l3d_get_matches_csr: no match result");
    cudaSetDevice(c->device);
    const long long rows = c->total_rows;
    if (rows == 0) { row_ptr_out[0] = 0; return 0; }
    int rc;
    L3D_RESERVE(c->d_rowptr, sizeof(long long) * (size_t)(rows + 1), "row_ptr");
    cub::TransformInputIterator<long long, CastI64, const int*> in((const int*)c->d_counts.p, CastI64());
    ScanTotal t;
    if ((rc = l3d_scan_total(c, in, (long long*)c->d_rowptr.p, rows, (const int*)c->d_counts.p, t, "row_ptr scan"))) return rc;
    c->launches += 2;   // cub: decoupled look-back init + scan kernels
    L3D_CUDA(c, cudaStreamSynchronize(c->stream), "sync");
    const long long total = t.last_out + t.last_src;
    L3D_CUDA(c, cudaMemcpyAsync((long long*)c->d_rowptr.p + rows, &total, sizeof(long long), cudaMemcpyHostToDevice, c->stream), "write total");
    L3D_RESERVE(c->d_csr, sizeof(l3d_match_rec) * (size_t)std::max<long long>(total, 1), "csr records");
    long long cells = rows * c->knn;
    k_compact_matches<<<(unsigned int)((cells + 255) / 256), 256, 0, c->stream>>>((const int*)c->d_counts.p, (const long long*)c->d_rowptr.p,
                                                                                   (const l3d_match_rec*)c->d_recs.p, c->knn, rows, (l3d_match_rec*)c->d_csr.p);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_compact_matches");
    L3D_CUDA(c, cudaMemcpyAsync(row_ptr_out, c->d_rowptr.p, sizeof(long long) * (rows + 1), cudaMemcpyDeviceToHost, c->stream), "download row_ptr");
    if (recs_out && total <= capacity && total > 0)
        L3D_CUDA(c, cudaMemcpyAsync(recs_out, c->d_csr.p, sizeof(l3d_match_rec) * (size_t)total, cudaMemcpyDeviceToHost, c->stream), "download records");
    L3D_CUDA(c, cudaStreamSynchronize(c->stream), "sync");
    return total;
}

// ------------------------------------------------------------------------------------------------ dense contract
// view pair (sv, tv) of the dense contract: its segments and cached rays, F (row-major, 9 floats), the camera centres and the outputs
static L3DDenseJob dense_job(const l3d_ctx* c, int sv, int tv, const float* F, float4* depths, float* overlaps, int rows_per_cta)
{
    const L3DViewDev& vs = c->h_views[sv]; const L3DViewDev& vt = c->h_views[tv];
    const float4* cache = (const float4*)c->d_cache.p;
    L3DDenseJob J = {c->segs() + vs.seg_off, c->segs() + vt.seg_off, cache + 3 * vs.seg_off, cache + 3 * vt.seg_off, depths, overlaps, {},
                     make_float3(vs.C[0], vs.C[1], vs.C[2]), make_float3(vt.C[0], vt.C[1], vt.C[2]), vs.nseg, vt.nseg, rows_per_cta,
                     (vt.nseg + DK_WARPS * DK_T * 32 - 1) / (DK_WARPS * DK_T * 32), 0};
    memcpy(J.F.m, F, sizeof(J.F.m));
    return J;
}

static int match_dense_impl(l3d_ctx* c, int sv, int tv, const float* F, float epi, float* depths, float* overlaps, int on_dev, bool filter)
{
    if (!c) return L3D_ERR_INVALID;
    if (!c->have_views) return l3d_fail(c, L3D_ERR_STATE, "l3d_match_dense: call l3d_set_views first");
    if (!F || !depths || !overlaps || sv < 0 || tv < 0 || sv >= c->num_views || tv >= c->num_views) return l3d_fail(c, L3D_ERR_INVALID, "l3d_match_dense: bad arguments");
    cudaSetDevice(c->device);
    const L3DViewDev& vs = c->h_views[sv]; const L3DViewDev& vt = c->h_views[tv];
    const int Ns = vs.nseg, Nt = vt.nseg;
    if (Ns == 0 || Nt == 0) return L3D_OK;
    const size_t cells = (size_t)Ns * Nt;
    float4* d_dep = (float4*)depths; float* d_ov = overlaps;
    HostBlock out[2] = {host_array(depths, sizeof(float4) * cells), host_array(overlaps, sizeof(float) * cells)};
    int rc;
    if (!on_dev) {
        if ((rc = l3d_stage_host(c, nullptr, 0, out, 2))) return rc;
        d_dep = (float4*)out[0].dev; d_ov = (float*)out[1].dev;
    }
    const L3DDenseJob J = dense_job(c, sv, tv, F, d_dep, d_ov, l3d_dense_rows_per_cta(Ns, Nt, c->num_sms));
    if (filter)
        k_match_dense<<<dim3(J.colb, (Ns + J.rows_per_cta - 1) / J.rows_per_cta), DK_THREADS, l3d_dense_smem_bytes(), c->stream>>>(J, epi);
    else
        k_match_dense_nofilter<<<dim3((Nt + DK_THREADS - 1) / DK_THREADS, (Ns + DKN_ROWS - 1) / DKN_ROWS), DK_THREADS, 0, c->stream>>>(J, epi);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_match_dense");
    if (!on_dev && (rc = l3d_unstage_host(c, out, 2, "sync"))) return rc;
    return L3D_OK;
}

int l3d_fp32_peak_probe(l3d_ctx* c, double* tflops_out)
{
    if (!c || !tflops_out) return L3D_ERR_INVALID;
    cudaSetDevice(c->device);
    int rc;
    L3D_RESERVE(c->cub_tmp, 256, "probe");      // result sink
    const int iters = 4096, blocks = c->num_sms * 8;
    ScopedEvent e0, e1;
    if ((rc = e0.create(c)) || (rc = e1.create(c))) return rc;
    double best = 0.0;
    for (int rep = 0; rep < 5; ++rep) {
        cudaEventRecord(e0.e, c->stream);
        k_fp32_peak<<<blocks, 256, 0, c->stream>>>((float*)c->cub_tmp.p, iters, 1.0000001f, 1e-9f);
        cudaEventRecord(e1.e, c->stream);
        ++c->launches;
        L3D_CUDA(c, cudaStreamSynchronize(c->stream), "k_fp32_peak");
        float ms = 0.f; cudaEventElapsedTime(&ms, e0.e, e1.e);
        double tf = 2.0 * 16.0 * iters * 256.0 * blocks / (ms * 1e-3) / 1e12;
        if (rep > 0 && tf > best) best = tf;
    }
    *tflops_out = best;
    return L3D_OK;
}

int l3d_match_dense(l3d_ctx* c, int sv, int tv, const float* F, float epi, float* depths, float* overlaps, int on_dev)
{ return match_dense_impl(c, sv, tv, F, epi, depths, overlaps, on_dev, true); }

// K_match_lines' dense device contract for MANY view pairs in ONE launch; outputs are device pointers, one pair of arrays per view pair
int l3d_match_dense_pairs(l3d_ctx* c, int npairs, const int32_t* pairs, const float* F, float epi, float* const* depths_dev, float* const* overlaps_dev)
{
    if (!c) return L3D_ERR_INVALID;
    if (!c->have_views) return l3d_fail(c, L3D_ERR_STATE, "l3d_match_dense_pairs: call l3d_set_views first");
    if (npairs < 0 || (npairs && (!pairs || !F || !depths_dev || !overlaps_dev))) return l3d_fail(c, L3D_ERR_INVALID, "l3d_match_dense_pairs: bad arguments");
    if (npairs == 0) return L3D_OK;
    cudaSetDevice(c->device);
    std::vector<L3DDenseJob> jobs;
    long long tiles = 0;
    for (int i = 0; i < npairs; ++i) {
        const int sv = pairs[2 * i], tv = pairs[2 * i + 1];
        if (sv < 0 || tv < 0 || sv >= c->num_views || tv >= c->num_views || !depths_dev[i] || !overlaps_dev[i]) return l3d_fail(c, L3D_ERR_INVALID, "l3d_match_dense_pairs: bad pair");
        if (c->h_views[sv].nseg == 0 || c->h_views[tv].nseg == 0) continue;
        // whole waves do not matter inside a batch: the tallest tile amortises the per-tile set-up best
        L3DDenseJob J = dense_job(c, sv, tv, F + 9 * (size_t)i, (float4*)depths_dev[i], overlaps_dev[i], DK_ROWS);
        J.tile0 = tiles;
        tiles += (long long)J.colb * ((J.Ns + DK_ROWS - 1) / DK_ROWS);
        jobs.push_back(J);
    }
    if (jobs.empty()) return L3D_OK;
    if (tiles >= (1ll << 31)) return l3d_fail(c, L3D_ERR_UNSUPPORTED, "l3d_match_dense_pairs: more than 2^31 tiles");
    int rc;
    L3D_RESERVE(c->d_dense_jobs, sizeof(L3DDenseJob) * jobs.size(), "dense jobs");
    L3D_CUDA(c, cudaMemcpyAsync(c->d_dense_jobs.p, jobs.data(), sizeof(L3DDenseJob) * jobs.size(), cudaMemcpyHostToDevice, c->stream), "dense jobs");
    L3D_CUDA(c, cudaStreamSynchronize(c->stream), "dense jobs");       // `jobs` is a local
    k_match_dense_batch<<<(unsigned int)tiles, DK_THREADS, l3d_dense_smem_bytes(), c->stream>>>((const L3DDenseJob*)c->d_dense_jobs.p, (int)jobs.size(), epi);
    ++c->launches;
    L3D_CUDA(c, cudaGetLastError(), "k_match_dense_batch");
    return L3D_OK;
}
int l3d_match_dense_nofilter(l3d_ctx* c, int sv, int tv, const float* F, float epi, float* depths, float* overlaps, int on_dev)
{ return match_dense_impl(c, sv, tv, F, epi, depths, overlaps, on_dev, false); }

} // extern "C"
