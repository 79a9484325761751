// l3d_collinear.cu — potentially collinear 2D segments within each view (SURVEY.md §8f-3).
//
// Replaces find_collinear_segments_GPU + K_collinearity (cudawrapper.cu:370-429, 689-705) and the host scan around it
// (View::findCollinGPU view.cc:173-209), or View::findCollinCPU (view.cc:212-263) under REF_CPU semantics.
// The reference fills a dense N x N char matrix per view (9 MB at N = 3000), copies it to the host and scans every row
// for ones.  Here ONE launch covers all views and emits the sparse answer directly: per segment the ascending list of
// its collinear segments (what collin_[i] holds after the host scan), as CSR over the global segment index.
//   pass 1 counts, a device scan turns counts into offsets, pass 2 re-evaluates and stores (the test is ~6 instructions
//   for 99.8 % of the cells, cheaper than keeping 1 bit per cell in HBM).
// A warp owns CL_RPW rows and walks the view's segments 32 at a time (coalesced float4 loads, L1-resident for the other
// warps of the CTA); ballot + popc keep every row's list in ascending order without atomics.
//
// ARITHMETIC (compiled with -fmad=false like the rest): collin_exact_f32 repeats K_collinearity's float operations in
// order; collin_exact_f64 repeats findCollinCPU (double geometry, float distances).  Both tests are symmetric in their
// two segments (the four on-segment tests are OR-ed, the distances max-ed), so evaluating (row, column) instead of the
// kernel's (max index, min index) gives the same bit.  The pre-filter only rejects cells whose FIRST point-to-line
// distance provably exceeds the threshold (0.01 % margin >> the 2^-23 rounding of the divide), which forces a zero.
#include "l3d_cub.cuh"

#define CL_WARPS 8
#define CL_RPW 4
#define CL_ROWS (CL_WARPS * CL_RPW)

// D_distance_p2l_2D_f3 (cudawrapper.cu:34-37)
__device__ __forceinline__ float cl_dist_f(float3 line, float px, float py)
{ return fabsf((line.x * px + line.y * py + line.z) / sqrtf(line.x * line.x + line.y * line.y)); }

__device__ __noinline__ bool collin_exact_f32(float4 p, float4 q, float dist_t)
{
    if (on_seg(p.x, p.y, p.z, p.w, q.x, q.y) || on_seg(p.x, p.y, p.z, p.w, q.z, q.w) || on_seg(q.x, q.y, q.z, q.w, p.x, p.y) ||
        on_seg(q.x, q.y, q.z, q.w, p.z, p.w))
        return false;                                                                   // overlap -> not collinear (cu:393-402)
    const float3 line1 = cross3(make_float3(p.x, p.y, 1.0f), make_float3(p.z, p.w, 1.0f));
    const float3 line2 = cross3(make_float3(q.x, q.y, 1.0f), make_float3(q.z, q.w, 1.0f));
    const float d1 = fmaxf(cl_dist_f(line1, q.x, q.y), cl_dist_f(line1, q.z, q.w));
    const float d2 = fmaxf(cl_dist_f(line2, p.x, p.y), cl_dist_f(line2, p.z, p.w));
    return fmaxf(d1, d2) < dist_t;
}

// View::pointOnSegment (view.cc:290-296), View::distance_point2line_2D (view.cc:266-269)
__device__ __forceinline__ bool cl_on_seg_d(double p1x, double p1y, double p2x, double p2y, double x, double y)
{ return ((p1x - x) * (p2x - x) + (p1y - y) * (p2y - y)) < 1e-12; }
__device__ __forceinline__ float cl_dist_d(double lx, double ly, double lz, double px, double py)
{ return (float)fabs((lx * px + ly * py + lz) / sqrtf((float)(lx * lx + ly * ly))); }

__device__ __noinline__ bool collin_exact_f64(float4 pf, float4 qf, float dist_t)
{
    const double p0x = pf.x, p0y = pf.y, p1x = pf.z, p1y = pf.w, q0x = qf.x, q0y = qf.y, q1x = qf.z, q1y = qf.w;
    if (cl_on_seg_d(p0x, p0y, p1x, p1y, q0x, q0y) || cl_on_seg_d(p0x, p0y, p1x, p1y, q1x, q1y) || cl_on_seg_d(q0x, q0y, q1x, q1y, p0x, p0y) ||
        cl_on_seg_d(q0x, q0y, q1x, q1y, p1x, p1y))
        return false;
    // Eigen cross of (x0,y0,1) x (x1,y1,1)
    const double l1x = p0y * 1.0 - 1.0 * p1y, l1y = 1.0 * p1x - p0x * 1.0, l1z = p0x * p1y - p0y * p1x;
    const double l2x = q0y * 1.0 - 1.0 * q1y, l2y = 1.0 * q1x - q0x * 1.0, l2z = q0x * q1y - q0y * q1x;
    const float d1 = fmaxf(cl_dist_d(l1x, l1y, l1z, q0x, q0y), cl_dist_d(l1x, l1y, l1z, q1x, q1y));
    const float d2 = fmaxf(cl_dist_d(l2x, l2y, l2z, p0x, p0y), cl_dist_d(l2x, l2y, l2z, p1x, p1y));
    return fmaxf(d1, d2) < dist_t;
}

// tiles[b] = (view, first row).  FILL = false: cnt[global seg] = list length.  FILL = true: idx[ptr[global seg] + i].
template <bool FILL, bool F64>
__global__ void __launch_bounds__(32 * CL_WARPS)
k_collinear(const float4* __restrict__ segs, const L3DViewDev* __restrict__ views, const int2* __restrict__ tiles, float dist_t,
            int* __restrict__ cnt, const long long* __restrict__ ptr, int* __restrict__ idx)
{
    const int2 tile = tiles[blockIdx.x];
    const L3DViewDev* V = views + tile.x;
    const int N = V->nseg, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float4* base = segs + V->seg_off;
    const int r0 = tile.y + warp * CL_RPW;
    if (r0 >= N) return;
    float4 p[CL_RPW];
    float lx[CL_RPW], ly[CL_RPW], lz[CL_RPW], thr[CL_RPW];           // float pre-filter: line through the row segment
    double dlx[CL_RPW], dly[CL_RPW], dlz[CL_RPW], dthr[CL_RPW];      // double pre-filter (REF_CPU)
    int count[CL_RPW];
    long long obase[CL_RPW];
#pragma unroll
    for (int i = 0; i < CL_RPW; ++i) {
        const int r = min(r0 + i, N - 1);
        p[i] = __ldg(base + r);
        count[i] = 0;
        obase[i] = FILL ? ptr[V->seg_off + r] : 0;
        if (F64) {
            const double x0 = p[i].x, y0 = p[i].y, x1 = p[i].z, y1 = p[i].w;
            dlx[i] = y0 * 1.0 - 1.0 * y1; dly[i] = 1.0 * x1 - x0 * 1.0; dlz[i] = x0 * y1 - y0 * x1;
            dthr[i] = (double)dist_t * (double)sqrtf((float)(dlx[i] * dlx[i] + dly[i] * dly[i])) * 1.0001;
        } else {
            const float3 l = cross3(make_float3(p[i].x, p[i].y, 1.0f), make_float3(p[i].z, p[i].w, 1.0f));
            lx[i] = l.x; ly[i] = l.y; lz[i] = l.z;
            thr[i] = dist_t * sqrtf(l.x * l.x + l.y * l.y) * 1.0001f;
        }
    }
    const unsigned int lt_mask = (1u << lane) - 1u;
    for (int c0 = 0; c0 < N; c0 += 32) {
        const int c = c0 + lane;
        const bool cv = c < N;
        const float4 q = __ldg(base + (cv ? c : 0));
#pragma unroll
        for (int i = 0; i < CL_RPW; ++i) {
            bool f = cv && (r0 + i) < N && c != r0 + i;
            if (f) {
                if (F64) {
                    const double a0 = dlx[i] * (double)q.x + dly[i] * (double)q.y + dlz[i];
                    f = !(fabs(a0) > dthr[i]) && collin_exact_f64(p[i], q, dist_t);
                } else {
                    const float a0 = lx[i] * q.x + ly[i] * q.y + lz[i];
                    f = !(fabsf(a0) > thr[i]) && collin_exact_f32(p[i], q, dist_t);
                }
            }
            const unsigned int b = __ballot_sync(0xffffffffu, f);
            if (FILL && f) idx[obase[i] + count[i] + __popc(b & lt_mask)] = c;
            count[i] += __popc(b);
        }
    }
    if (!FILL && lane == 0) {
#pragma unroll
        for (int i = 0; i < CL_RPW; ++i)
            if (r0 + i < N) cnt[V->seg_off + r0 + i] = count[i];
    }
}

extern "C" {

// Collinear segments of every view (Line3D::findCollinearSegments line3D.cc:1827-1849 over View::findCollinearSegments
// view.cc:152-171).  dist_t <= 1e-12 switches the collinearity links off again.  semantics: L3D_SEM_REF_GPU (float, as
// K_collinearity) or L3D_SEM_REF_CPU (findCollinCPU).  The lists stay on the device for l3d_affinity_matrix /
// l3d_affinity_edges; l3d_get_collinear downloads them.
int l3d_find_collinear(l3d_ctx* c, float dist_t, int semantics)
{
    if (!c) return L3D_ERR_INVALID;
    CollinState& K = c->collin;
    const bool off = !(dist_t > 1e-12f);
    const bool sem_ok = semantics == L3D_SEM_REF_GPU || semantics == L3D_SEM_REF_CPU;
    // already off, or already computed (view.cc:154-158): the lists and the affinity matrix built on them stay
    const bool unchanged = sem_ok && (off ? !K.valid : K.valid && K.dist_t == dist_t && K.sem == semantics);
    if (!unchanged) c->drop(Stage::Collinear);
    if (!c->have_views) return l3d_fail(c, L3D_ERR_STATE, "l3d_find_collinear: call l3d_set_views first");
    if (!sem_ok) return l3d_fail(c, L3D_ERR_INVALID, "l3d_find_collinear: bad semantics");
    if (off || unchanged) return L3D_OK;
    cudaSetDevice(c->device);
    const long long N = c->total_segs;
    if (N == 0) { K.total = 0; K.valid = true; K.dist_t = dist_t; K.sem = semantics; return L3D_OK; }
    std::vector<int2> tiles;
    for (int v = 0; v < c->num_views; ++v)
        for (int r = 0; r < c->h_views[v].nseg; r += CL_ROWS) tiles.push_back(make_int2(v, r));
    int rc;
    L3D_RESERVE(K.d_tiles, sizeof(int2) * tiles.size(), "collinear tiles");
    L3D_RESERVE(K.d_cnt, 4 * (N + 1), "collinear counts"); L3D_RESERVE(K.d_ptr, 8 * (N + 1), "collinear offsets");
    cudaStream_t st = c->stream;
    L3D_CUDA(c, cudaMemcpyAsync(K.d_tiles.p, tiles.data(), sizeof(int2) * tiles.size(), cudaMemcpyHostToDevice, st), "collinear tiles");
    L3D_CUDA(c, cudaMemsetAsync(K.d_cnt.p, 0, 4 * (size_t)(N + 1), st), "collinear counts");
    const unsigned int nb = (unsigned int)tiles.size();
    if (semantics == L3D_SEM_REF_CPU)
        k_collinear<false, true><<<nb, 32 * CL_WARPS, 0, st>>>(c->segs(), c->views(), (const int2*)K.d_tiles.p, dist_t, (int*)K.d_cnt.p, nullptr, nullptr);
    else
        k_collinear<false, false><<<nb, 32 * CL_WARPS, 0, st>>>(c->segs(), c->views(), (const int2*)K.d_tiles.p, dist_t, (int*)K.d_cnt.p, nullptr, nullptr);
    if ((rc = l3d_cub(c, "collinear scan", [&](void* tmp, size_t& bytes) {
             return cub::DeviceScan::ExclusiveSum(tmp, bytes, (const int*)K.d_cnt.p, (long long*)K.d_ptr.p, N + 1, st); }))) return rc;
    long long total = 0;
    L3D_CUDA(c, cudaMemcpyAsync(&total, (long long*)K.d_ptr.p + N, 8, cudaMemcpyDeviceToHost, st), "collinear total");
    L3D_CUDA(c, cudaStreamSynchronize(st), "collinear count");
    L3D_RESERVE(K.d_idx, 4 * total, "collinear lists");
    if (total > 0) {
        if (semantics == L3D_SEM_REF_CPU)
            k_collinear<true, true><<<nb, 32 * CL_WARPS, 0, st>>>(c->segs(), c->views(), (const int2*)K.d_tiles.p, dist_t, nullptr, (const long long*)K.d_ptr.p, (int*)K.d_idx.p);
        else
            k_collinear<true, false><<<nb, 32 * CL_WARPS, 0, st>>>(c->segs(), c->views(), (const int2*)K.d_tiles.p, dist_t, nullptr, (const long long*)K.d_ptr.p, (int*)K.d_idx.p);
    }
    c->launches += total > 0 ? 4 : 3;
    L3D_CUDA(c, cudaGetLastError(), "k_collinear");
    K.total = total; K.valid = true; K.dist_t = dist_t; K.sem = semantics;
    return L3D_OK;
}

long long l3d_collinear_total(const l3d_ctx* c) { return (c && c->collin.valid) ? c->collin.total : 0; }

// collin_ of one view (view.h) as CSR: row_ptr_out[nseg + 1] (relative to the view), idx_out = segment ids, ascending per
// row.  Returns the number of entries of the view (even if > cap; then only row_ptr_out is filled).
long long l3d_get_collinear(l3d_ctx* c, int view, long long* row_ptr_out, int32_t* idx_out, long long cap)
{
    if (!c) return L3D_ERR_INVALID;
    if (!c->collin.valid) return l3d_fail(c, L3D_ERR_STATE, "l3d_get_collinear: call l3d_find_collinear first");
    if (view < 0 || view >= c->num_views) return l3d_fail(c, L3D_ERR_INVALID, "l3d_get_collinear: bad view");
    cudaSetDevice(c->device);
    const L3DViewDev& V = c->h_views[view];
    if (V.nseg == 0) { if (row_ptr_out) row_ptr_out[0] = 0; return 0; }
    std::vector<long long> ptr((size_t)V.nseg + 1);
    L3D_CUDA(c, cudaMemcpyAsync(ptr.data(), (const long long*)c->collin.d_ptr.p + V.seg_off, 8 * ((size_t)V.nseg + 1), cudaMemcpyDeviceToHost, c->stream), "download collinear offsets");
    L3D_CUDA(c, cudaStreamSynchronize(c->stream), "sync");
    const long long first = ptr[0], n = ptr[V.nseg] - first;
    if (row_ptr_out) for (int i = 0; i <= V.nseg; ++i) row_ptr_out[i] = ptr[i] - first;
    if (idx_out && n > 0 && n <= cap) {
        L3D_CUDA(c, cudaMemcpyAsync(idx_out, (const int*)c->collin.d_idx.p + first, 4 * (size_t)n, cudaMemcpyDeviceToHost, c->stream), "download collinear lists");
        L3D_CUDA(c, cudaStreamSynchronize(c->stream), "sync");
    }
    return n;
}

}  // extern "C"
